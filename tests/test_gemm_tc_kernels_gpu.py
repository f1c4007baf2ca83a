"""GPU: the tensor-core dense GEMM gemm_tc_kernel<BLOCK_N, A_MN, B_MN, kStages, EPI, SPLIT> (csrc/gemm_tc.cu) and its
split-K reduce in isolation, through the three C entry points that reach them: tb_gemm_bf16_tn, tb_gemm_bf16_ex and
tb_gemm_bf16x3_ex.  Layouts: "kk" forward (A [M, K], B [N, K]), "km" input gradient (B stored [K, N]), "mm" weight
gradient (A stored [K, M], B [K, N]).

- Instantiations.  The build holds 42; these entry points reach 31, and every case below is named by the one it must
  run.  The launch rules (gemm_block_n, gemm_stages and the EPI selection) are restated here, and one profiler pass
  checks the demangled name of every launch:
  - SPLIT (split-bf16 operands, tb_gemm_bf16x3_ex), 21: kk at BLOCK_N 32 / 64 / 128, km and mm at 64 / 128, each at
    EPI 0, 1 and 2;
  - single-plane EPI 0 (tb_gemm_bf16_ex), 7: the same seven layouts;
  - single-plane EPI 1 (tb_gemm_bf16_tn), 3: kk at 32 / 64 / 128.
  The other 11 need a TcEpilogue that none of these entry points builds; the network tests at precision bf16
  (test_resnet_width_gpu.py, test_resnet_obs_gpu.py) run them:
  - single-plane EPI 1 with an MN-major B (km and mm at 64 / 128), e.g. a ResNet bf16 weight gradient with one split;
  - single-plane EPI 2 (all seven layouts), the ResNet bf16 residual addend16.
- Exact.  The hi and lo planes hold independent small integers (hi in [-8, 8], lo in [-4, 4]), the bias integers and
  the scale a power of two, K <= 20000: every partial sum stays below 2^24, so fp32 accumulation in any order is
  exact.  C must equal hi.hi + hi.lo + lo.hi (no lo.lo) in float64, and the bf16 output the round-to-nearest-even hi /
  lo split of it (single-plane: the hi part of the exact hi.hi product).  Zeros of either sign compare equal.  Every
  reachable instantiation runs at M in {1, 2, 127, 128, 129, 385, 2592}, N tails, K not a multiple of 64, and on a
  persistent grid with more work items than CTAs (some CTAs take three).
- Bounded.  randn operands split with tests/sw_image.py's `split`, against float64 on the hi + lo values within
  `sw_image.tolerance` (single-plane: lolo=False); each case shows the reference with one lo product left out
  (single-plane: one 64-term k-block left out) at least ten times outside the bound.
- Split-K (splits 2, 3, 7; trailing empty splits; more splits than k-blocks): the reduce applies scale, then bias, then
  ReLU, exactly; a partial buffer of exactly splits * M * roundup(N, 32) floats prefilled with NaN gives the bits of a
  zeroed one.
- Epilogue branches.  The kernel takes a vector or a scalar path from N, the leading dimensions and the alignment of
  C, C16, bias and mask; the same call with each of those moved off alignment gives the same bits, and a bf16 mask
  keeps an element exactly where it is > 0 (not where it is +0, -0, negative or NaN) on both paths.
- Memory.  Every output and partial buffer sits between 64 guard bytes that must come back untouched, outputs are
  prefilled with 0xFF bytes, the columns in [N, ldc) keep them, and calls with M = 0 or N = 0 write nothing."""
import re

import pytest
import torch

from tests import sw_image as S
from tests.test_gemm_dense_tiles_gpu import block_n

pytestmark = pytest.mark.gpu

GUARD = 64
LAYOUTS = {"kk": (False, False), "km": (False, True), "mm": (True, True)}
BF16 = torch.bfloat16
MASK_SPECIALS = [0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x7F80, 0xFF80, 0x7FC0, 0xFFC0, 0x7F81, 0x7F7F, 0x3F80]


# ---- launch rules (csrc/gemm_tc.cu), restated -------------------------------------------------------------------------
def stages(bn, split):
    """gemm_stages: the deepest ring of at most 4 stages beside the staging tiles in 227 KB - split operands 4 at
    BLOCK_N 32 / 64 and 3 at 128, single-plane 4 everywhere"""
    return 3 if split and bn == 128 else 4


def epi_of(mask=False, bias=False, relu=False, scale=1.0, splits=1):
    """EPI: 2 with a mask or addend, 1 with bias, ReLU or scale != 1 and no partial buffer, else 0"""
    if mask:
        return 2
    return 1 if (bias or relu or scale != 1.0) and splits == 1 else 0


def kname(inst):
    bn, lay, epi, split = inst
    tf = lambda b: "true" if b else "false"
    a_mn, b_mn = LAYOUTS[lay]
    return "gemm_tc_kernel<%d, %s, %s, %d, %d, %s>" % (bn, tf(a_mn), tf(b_mn), stages(bn, split), epi, tf(split))


def inst_id(inst):
    bn, lay, epi, split = inst
    return "%s%d-epi%d-%s" % (lay, bn, epi, "x3" if split else "bf16")


BNS = {"kk": (32, 64, 128), "km": (64, 128), "mm": (64, 128)}
INSTS = ([(bn, lay, e, True) for lay in LAYOUTS for bn in BNS[lay] for e in (0, 1, 2)]
         + [(bn, lay, 0, False) for lay in LAYOUTS for bn in BNS[lay]]
         + [(bn, "kk", 1, False) for bn in BNS["kk"]])

MS = [1, 2, 127, 128, 129, 385, 2592]
NS = [24, 519, 17, 50, 520, 32, 8520, 130, 8000, 4000]
KS = [200, 72, 1, 136, 520, 1000, 63]
GRID = [(40000, 24), (4100, 520), (8960, 640)]   # more work items than the 132 CTAs: 313, 297, 350


def items(M, N, splits, bn):
    return -(-M // 128) * -(-N // bn) * splits


def shapes(inst):
    """(M, N, K) of the exact sweep: each M with the first N of NS (rotated by the M's index) that gives the
    instantiation's BLOCK_N, then one GRID shape"""
    bn, lay, _, _ = inst
    b_mn = LAYOUTS[lay][1]
    out = []
    for i, M in enumerate(MS):
        N = next(n for n in NS[i:] + NS[:i] if block_n(M, n, 1, b_mn) == bn)
        out.append((M, N, KS[i]))
    out.append(next((M, N, 100) for M, N in GRID if block_n(M, N, 1, b_mn) == bn))
    return out


EXACT = [(inst, M, N, K) for inst in INSTS for (M, N, K) in shapes(inst)]


# ---- C calls and guarded buffers -------------------------------------------------------------------------------------
def lib():
    from torchbeast_b200 import _lib
    return _lib.lib()


def stream():
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def call(name, *args):
    rc = getattr(lib(), name)(*args)
    assert rc == 0, "%s: %s" % (name, lib().tb_last_error().decode())


def rup(n, m):
    return -(-n // m) * m


class Buf:
    """n elements of dtype `off` elements past 64 guard bytes (random) and followed by 64 more; prefilled with 0xFF
    bytes, or with `values`"""

    def __init__(self, n, dtype=torch.float32, off=0, values=None):
        es = torch.empty(0, dtype=dtype).element_size()
        self.lo, self.hi = GUARD + off * es, GUARD + (off + n) * es
        self.raw = torch.randint(0, 256, (self.hi + GUARD,), dtype=torch.uint8, device="cuda")
        self.raw[GUARD:self.hi] = 255
        self.t = self.raw[self.lo:self.hi].view(dtype)
        if values is not None:
            self.t.copy_(values.reshape(-1))
        self.init = self.raw.clone()

    @property
    def ptr(self):
        import ctypes
        return ctypes.c_void_p(self.raw.data_ptr() + self.lo)

    def guards_intact(self):
        return torch.equal(self.raw[:GUARD], self.init[:GUARD]) and torch.equal(self.raw[self.hi:], self.init[self.hi:])

    def unchanged(self):
        return torch.equal(self.raw, self.init)


def ptr(b):
    return None if b is None else b.ptr


def canon(t):
    """integer image of a float32 / bf16 tensor with -0 folded into +0"""
    return (t + 0).view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def same(got, want):
    return torch.equal(canon(got), canon(want))


class Operands:
    """A and B of one call in their stored layouts, [planes, rows, ld] bf16 with NaN in the padding columns, and their
    float64 values as math operands A [M, K], B [N, K] (hi, lo; lo is None for single-plane operands).
    exact: hi integers in [-8, 8], lo in [-4, 4]; else randn split into hi / lo (or rounded to bf16)."""

    def __init__(self, lay, split, M, N, K, seed, exact):
        g = torch.Generator(device="cuda").manual_seed(seed)
        a_mn, b_mn = LAYOUTS[lay]
        self.a_mn, self.b_mn = a_mn, b_mn
        self.A, self.lda, self.a_lo, (self.Ah, self.Al) = self._make((K, M) if a_mn else (M, K), a_mn, split, g, exact)
        self.B, self.ldb, self.b_lo, (self.Bh, self.Bl) = self._make((K, N) if b_mn else (N, K), b_mn, split, g, exact)

    @staticmethod
    def _make(shape, mn, split, g, exact):
        rows, cols = shape
        ld = rup(cols, 8)
        npl = 2 if split else 1
        buf = torch.full((npl, rows, ld), float("nan"), dtype=BF16, device="cuda")
        if exact:
            buf[0, :, :cols] = torch.randint(-8, 9, shape, device="cuda", generator=g).to(BF16)
            if split:
                buf[1, :, :cols] = torch.randint(-4, 5, shape, device="cuda", generator=g).to(BF16)
        else:
            x = torch.randn(shape, device="cuda", generator=g)
            hi, lo = S.split(x)
            buf[0, :, :cols] = hi
            if split:
                buf[1, :, :cols] = lo
        math = [buf[p, :, :cols].double() for p in range(npl)]
        math = [m.t() if mn else m for m in math] + ([None] if npl == 1 else [])
        return buf, ld, (rows * ld if split else 0), math

    def acc(self, drop=None):
        """float64 hi.hi + hi.lo + lo.hi; drop="lo" leaves out lo(A).hi(B), drop="kblock" the first 64 k terms"""
        acc = self.Ah @ self.Bh.t()
        if self.Al is not None:
            acc = acc + self.Ah @ self.Bl.t() + (0 if drop == "lo" else self.Al @ self.Bh.t())
        if drop == "kblock":
            acc = acc - self.Ah[:, :64] @ self.Bh[:, :64].t()
        return acc


def epilogue_ref(acc, scale=1.0, bias=None, relu=0, mask=None):
    """scale, then bias, then ReLU, then the mask (kept where the bf16 mask is > 0)"""
    out = acc * scale
    if bias is not None:
        out = out + bias.double()
    if relu:
        out = out.clamp_min(0)
    if mask is not None:
        out = torch.where(mask.double() > 0, out, torch.zeros_like(out))
    return out


def launch(inst, ops, M, N, K, C=None, ldc=0, C16=None, ldc16=0, c16_lo=0, bias=None, scale=1.0, relu=0, mask=None,
           ldmask=0, splits=1, partial=None):
    """one call through the entry point that reaches `inst`"""
    _, _, epi, split = inst
    if split:
        call("tb_gemm_bf16x3_ex", ops.A.data_ptr(), ops.B.data_ptr(), M, N, K, ops.lda, ops.ldb, int(ops.a_mn),
             int(ops.b_mn), ops.a_lo, ops.b_lo, ptr(C), ldc, ptr(C16), ldc16, c16_lo, ptr(bias), scale, relu, ptr(mask),
             ldmask, splits, ptr(partial), stream())
    elif epi == 1 or C16 is not None:
        assert not ops.a_mn and not ops.b_mn and splits == 1
        call("tb_gemm_bf16_tn", ops.A.data_ptr(), ops.B.data_ptr(), M, N, K, ops.lda, ops.ldb, ptr(C), ldc, ptr(C16),
             ldc16, ptr(bias), scale, relu, stream())
    else:
        assert bias is None and scale == 1.0 and not relu
        call("tb_gemm_bf16_ex", ops.A.data_ptr(), ops.B.data_ptr(), M, N, K, ops.lda, ops.ldb, int(ops.a_mn),
             int(ops.b_mn), ptr(C), ldc, splits, ptr(partial), stream())


def epilogue_inputs(inst, M, N, seed, exact):
    """(bias values, scale, relu, mask values [M, N] bf16) for the instantiation's EPI"""
    _, _, epi, _ = inst
    if epi == 0:
        return None, 1.0, 0, None
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    bias = (torch.randint(-64, 65, (N,), device="cuda", generator=g).float() if exact
            else torch.randn(N, device="cuda", generator=g))
    mask = None
    if epi == 2:
        mask = torch.randn(M, N, device="cuda", generator=g).to(BF16)
        mask[:, :min(N, len(MASK_SPECIALS))] = special_mask(min(N, len(MASK_SPECIALS)))
    return bias, (0.5 if exact else 0.75), 1, mask


def special_mask(n):
    return torch.tensor(MASK_SPECIALS[:n], dtype=torch.int32).to(torch.int16).view(BF16).cuda()


def run(inst, ops, M, N, K, bias, scale, relu, mask, want_c=True, planes16=None, c_off=0, ldc=None, c16_off=0,
        ldc16=None, bias_off=0, mask_off=0, ldmask=None):
    """launch `inst` with guarded outputs; planes16: bf16 output planes (0, 1 = hi, 2 = hi and lo; default: all the
    entry point writes).  Returns (C [M, ldc] or None, hi [M, ldc16] or None, lo [M, ldc16] or None)."""
    _, _, epi, split = inst
    if planes16 is None:
        planes16 = 2 if split else int(epi == 1)
    ldc = ldc or rup(N, 8) + 8
    ldc16 = ldc16 or rup(N, 8) + 8
    C = Buf(M * ldc, off=c_off) if want_c else None
    c16_lo = rup(M * ldc16, 8) if planes16 == 2 else 0
    C16 = Buf(c16_lo + M * ldc16, BF16, off=c16_off) if planes16 else None
    b = Buf(N, off=bias_off, values=bias) if bias is not None else None
    m = None
    if mask is not None:
        ldmask = ldmask or rup(N, 8)
        full = torch.full((M, ldmask), float("nan"), dtype=BF16, device="cuda")
        full[:, :N] = mask
        m = Buf(M * ldmask, BF16, off=mask_off, values=full)
    launch(inst, ops, M, N, K, C, ldc, C16, ldc16, c16_lo, b, scale, relu, m, ldmask or 0)
    torch.cuda.synchronize()
    for buf in (C, C16, b, m):
        assert buf is None or buf.guards_intact()
    for buf in (b, m):
        assert buf is None or buf.unchanged()
    c = C.t.view(M, ldc) if C else None
    if c is not None:  # the columns in [N, ldc) keep their 0xFF bytes
        assert bool((c[:, N:].view(torch.int32) == -1).all())
    hi = lo = None
    if C16:
        hi = C16.t[:M * ldc16].view(M, ldc16)
        lo = C16.t[c16_lo:c16_lo + M * ldc16].view(M, ldc16) if c16_lo else None
        for t in (hi, lo):
            assert t is None or bool((t[:, N:].view(torch.int16) == -1).all())
    return c, hi, lo


def check_bf16_planes(hi, lo, value, N):
    """hi (and lo) = the round-to-nearest-even split of the float32 value, bit for bit"""
    want_hi, want_lo = S.split(value)
    assert same(hi[:, :N], want_hi), "bf16 hi plane"
    if lo is not None:
        assert same(lo[:, :N], want_lo), "bf16 lo plane"


# ---- instantiations --------------------------------------------------------------------------------------------------
def test_case_table_covers_the_reachable_instantiations():
    assert len(INSTS) == len(set(INSTS)) == 31 and len({kname(i) for i in INSTS}) == 31
    assert [stages(bn, True) for bn in (32, 64, 128)] == [4, 4, 3] and {stages(bn, False) for bn in (32, 64, 128)} == {4}
    assert epi_of(mask=True) == 2 and epi_of(bias=True) == epi_of(relu=True) == epi_of(scale=0.5) == 1
    assert epi_of(bias=True, scale=0.5, relu=True, splits=3) == 0 and epi_of() == 0
    for inst in INSTS:
        sh = shapes(inst)
        assert [M for M, _, _ in sh[:len(MS)]] == MS
        assert any(K % 64 for _, _, K in sh)
        counts = [items(M, N, 1, inst[0]) for M, N, _ in sh]
        assert min(counts) < 132 and max(counts) > 2 * 132, (inst, counts)  # a grid with 3-item CTAs
    assert {N for inst in INSTS for _, N, _ in shapes(inst)} >= {17, 24, 32, 50, 519, 520}


def _launch_plan():
    """(function, expected kernel names) for the first exact shape of every instantiation and each split-K case"""
    plan = []
    for inst in INSTS:
        M, N, K = shapes(inst)[0]
        ops = Operands(inst[1], inst[3], M, N, K, 1, exact=True)
        bias, scale, relu, mask = epilogue_inputs(inst, M, N, 1, exact=True)
        assert epi_of(mask is not None, bias is not None, relu, scale) == inst[2]
        plan.append((lambda inst=inst, ops=ops, a=(M, N, K, bias, scale, relu, mask): run(inst, ops, *a), [kname(inst)]))
    for lay, split, M, N, K, splits in SPLITK:
        inst = (block_n(M, N, splits, lay != "kk"), lay, 0, split)
        plan.append((lambda a=(lay, split, M, N, K, splits): splitk(*a, epilogue=True), [kname(inst), "splitk_reduce_kernel"]))
    return plan


def _short(name):
    """'void tb::(anonymous namespace)::gemm_tc_kernel<(int)64, (bool)0, ...>(...)' -> 'gemm_tc_kernel<64, false, ...>'"""
    m = re.search(r"\b(gemm_tc_kernel|splitk_reduce_kernel)\b(<[^>]*>)?", name)
    if not m:
        return None
    args = (m.group(2) or "").replace("(bool)0", "false").replace("(bool)1", "true").replace("(int)", "")
    return m.group(1) + re.sub(r"\s*,\s*", ", ", args)


def test_every_launch_runs_the_expected_instantiation():
    from torch.profiler import ProfilerActivity, profile
    plan = _launch_plan()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn, _ in plan:
            fn()
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    if not kernels:
        pytest.skip("the profiler recorded no CUDA kernel activity on this machine")
    got = [s for s in (_short(e.name) for e in sorted(kernels, key=lambda e: e.time_range.start)) if s]
    want = [n for _, names in plan for n in names]
    assert len(got) == len(want), (len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "launch %d: ran %s, expected %s" % (i, g, w)


# ---- exact integer products ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inst,M,N,K", EXACT, ids=["%s-%dx%dx%d" % ((inst_id(c[0]),) + c[1:]) for c in EXACT])
def test_exact(inst, M, N, K):
    bn, lay, epi, split = inst
    assert block_n(M, N, 1, lay != "kk") == bn
    seed = M * 7 + N * 3 + K
    ops = Operands(lay, split, M, N, K, seed, exact=True)
    bias, scale, relu, mask = epilogue_inputs(inst, M, N, seed, exact=True)
    C, hi, lo = run(inst, ops, M, N, K, bias, scale, relu, mask)
    ref = epilogue_ref(ops.acc(), scale, bias, relu, mask)
    assert bool((ref.abs() < 2 ** 24).all())
    assert same(C[:, :N], ref.float()), "C differs from the exact product"
    if hi is not None:
        check_bf16_planes(hi, lo, ref.float(), N)


# ---- bounded randn products ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inst", INSTS, ids=[inst_id(i) for i in INSTS])
def test_bounded(inst):
    """randn operands at M = 2592 (the learner's T * B) and K = 3000 within sw_image.tolerance; the reference with one
    lo product (single-plane: one 64-term k-block) left out is at least ten times outside it; two runs agree bit for
    bit and the bf16 output is the split (single-plane: the rounding) of C"""
    bn, lay, epi, split = inst
    M, N, K = 2592, shapes(inst)[-2][1], 3000
    assert block_n(M, N, 1, lay != "kk") == bn
    ops = Operands(lay, split, M, N, K, 17 + bn, exact=False)
    bias, scale, relu, mask = epilogue_inputs(inst, M, N, 17 + bn, exact=False)
    C, hi, lo = run(inst, ops, M, N, K, bias, scale, relu, mask)
    C2, hi2, lo2 = run(inst, ops, M, N, K, bias, scale, relu, mask)
    assert torch.equal(C.view(torch.int32), C2.view(torch.int32)), "two runs differ"
    c = C[:, :N]
    ref = epilogue_ref(ops.acc(), scale, bias, relu, mask)
    drop = epilogue_ref(ops.acc("lo" if split else "kblock"), scale, bias, relu, mask)
    A = ops.Ah + (ops.Al if split else 0)
    B = ops.Bh + (ops.Bl if split else 0)
    tol = S.tolerance(K, S.rms(A) * S.rms(B) * scale, ref, extra=bias.double() if bias is not None else None, lolo=split)
    assert torch.isfinite(c).all()
    err, miss = S.excess(c, ref, tol), S.excess(drop, ref, tol)
    print("bounded %s: error / bound %.3g, dropped %s / bound %.3g" % (inst_id(inst), err, "lo" if split else "k-block", miss))
    assert err <= 1.0, "max |err| / tol = %.3g" % err
    assert miss >= 10.0, "the reference with a term left out is only %.3g x the bound" % miss
    if hi is not None:
        assert torch.equal(hi.view(torch.int16), hi2.view(torch.int16))
        check_bf16_planes(hi, lo, c, N)


# ---- split-K ---------------------------------------------------------------------------------------------------------
SPLITK = [  # layout, split operands, M, N, K, splits
    ("mm", True, 300, 519, 1000, 2),
    ("km", True, 129, 50, 700, 3),
    ("mm", True, 2592, 520, 2592, 7),
    ("km", True, 1, 24, 300, 7),
    ("mm", True, 385, 130, 200, 3),      # 4 k-blocks, 2 per split: split 2 is empty
    ("km", True, 128, 519, 100, 7),      # 2 k-blocks over 7 splits: 5 empty
    ("kk", True, 200, 130, 20000, 3),    # the longest exact K
    ("mm", False, 2076, 520, 2592, 7),
    ("km", False, 127, 519, 200, 3),
    ("mm", False, 129, 50, 100, 7),
]


def splitk(lay, split, M, N, K, splits, epilogue, stale=True):
    """one split-K call (split operands with scale 0.5, integer bias and ReLU applied by the reduce when `epilogue`);
    returns (C [M, ldc], expected, partial Buf)"""
    ops = Operands(lay, split, M, N, K, M + N + K + splits, exact=True)
    inst = (block_n(M, N, splits, lay != "kk"), lay, 0, split)
    bias, scale, relu = None, 1.0, 0
    if epilogue and split:
        bias = torch.randint(-64, 65, (N,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(K)).float()
        scale, relu = 0.5, 1
    ldc = rup(N, 8) + 8
    C = Buf(M * ldc)
    part = Buf(splits * M * rup(N, 32))
    if not stale:
        part.t.zero_()
        part.init = part.raw.clone()
    b = Buf(N, values=bias) if bias is not None else None
    launch(inst, ops, M, N, K, C, ldc, bias=b, scale=scale, relu=relu, splits=splits, partial=part)
    return C, ldc, epilogue_ref(ops.acc(), scale, bias, relu), part


@pytest.mark.parametrize("lay,split,M,N,K,splits", SPLITK)
def test_split_k_exact(lay, split, M, N, K, splits):
    torch.cuda.synchronize()
    C, ldc, ref, part = splitk(lay, split, M, N, K, splits, epilogue=True)
    C0, _, _, part0 = splitk(lay, split, M, N, K, splits, epilogue=True, stale=False)
    torch.cuda.synchronize()
    for b in (C, part, C0, part0):
        assert b.guards_intact()
    c = C.t.view(M, ldc)
    assert bool((c[:, N:].view(torch.int32) == -1).all())
    assert same(c[:, :N], ref.float()), "split-K result differs from the exact product"
    assert torch.equal(C.t.view(torch.int32), C0.t.view(torch.int32)), "a NaN partial buffer changed the result"


# ---- epilogue branches -----------------------------------------------------------------------------------------------
VARIANTS = {  # the layout of the output side, all else equal: aligned and contiguous, then one thing moved off it
    "aligned": {},
    "c_off": dict(c_off=1, ldc=1),
    "c16_off": dict(c16_off=1, ldc16=1),
    "bias_off": dict(bias_off=1),
    "mask_off": dict(mask_off=3, ldmask=3),
}
BRANCH_INSTS = [(64, "kk", 2, True), (64, "km", 2, True), (64, "kk", 1, True), (64, "kk", 1, False)]


@pytest.mark.parametrize("planes16", [0, 1, 2], ids=["C", "C16", "C16+lo"])
@pytest.mark.parametrize("inst", BRANCH_INSTS, ids=[inst_id(i) for i in BRANCH_INSTS])
def test_epilogue_branches_give_the_same_bits(inst, planes16):
    """M = 300, N = 520 (BLOCK_N 64): 16 full 32-column chunks and a tail chunk of 8 columns per row.  The mask holds
    +-0, subnormals, +-inf, NaN of both signs, the largest finite value and 1 in a full chunk (columns 0-11) and in the
    tail chunk (512-519).  Offsets are in elements; ldc / ldc16 / ldmask are N plus the variant's value."""
    bn, lay, epi, split = inst
    if planes16 == 2 and not split:
        pytest.skip("a single-plane product has no lo plane to write")
    M, N, K = 300, 520, 200
    assert block_n(M, N, 1, lay != "kk") == bn
    ops = Operands(lay, split, M, N, K, 5, exact=True)
    bias, scale, relu, mask = epilogue_inputs(inst, M, N, 5, exact=True)
    if mask is not None:
        mask[:, 512:520] = special_mask(8)
    ref = epilogue_ref(ops.acc(), scale, bias, relu, mask).float()
    results = {}
    for name, var in VARIANTS.items():
        if name == "mask_off" and mask is None:
            continue
        kw = dict(var)
        for ld in ("ldc", "ldc16", "ldmask"):
            kw[ld] = N + kw.get(ld, 0)
        C, hi, lo = run(inst, ops, M, N, K, bias, scale, relu, mask, want_c=planes16 == 0, planes16=planes16, **kw)
        if C is not None:
            assert same(C[:, :N], ref), "%s: C differs from the exact result" % name
            results[name] = [C[:, :N].view(torch.int32)]
        else:
            check_bf16_planes(hi, lo, ref, N)
            results[name] = [t[:, :N].view(torch.int16) for t in (hi, lo) if t is not None]
    base = results.pop("aligned")
    for name, got in results.items():
        assert len(got) == len(base) and all(torch.equal(a, b) for a, b in zip(got, base)), name


# ---- empty sizes -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N", [(0, 40), (40, 0)])
@pytest.mark.parametrize("inst,splits", [((64, "kk", 2, True), 1), ((64, "mm", 0, True), 3), ((32, "kk", 1, False), 1),
                                         ((64, "km", 0, False), 3)], ids=["x3-mask", "x3-splitk", "tn", "ex-splitk"])
def test_empty_sizes_write_nothing(inst, splits, M, N):
    bn, lay, epi, split = inst
    ops = Operands(lay, split, max(M, 1), max(N, 1), 64, 3, exact=True)
    C, C16, part = Buf(64 * 64), Buf(2 * 64 * 64, BF16), Buf(3 * 64 * 64)
    bias = Buf(64, values=torch.zeros(64, device="cuda")) if epi else None
    mask = Buf(64 * 64, BF16, values=torch.ones(64 * 64, device="cuda")) if epi == 2 else None
    with16 = splits == 1 and (split or epi == 1)
    launch(inst, ops, M, N, 64, C, 64, C16 if with16 else None, 64, 64 * 64 if split and with16 else 0, bias,
           0.5 if epi else 1.0, 0, mask, 64, splits, part if splits > 1 else None)
    torch.cuda.synchronize()
    assert C.unchanged() and C16.unchanged() and part.unchanged()


# ---- tb_f32_to_bf16 --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,ld,ld16", [(37, 519, 519, 520), (5, 3, 7, 8), (600, 1000, 1003, 1008)])
def test_f32_to_bf16_rounds_to_nearest_even(rows, cols, ld, ld16):
    """bit for bit torch's round-to-nearest-even (any NaN for NaN), padding columns [cols, ld16) zero; 600 x 1008 is
    past the kernel's grid cap of 132 * 16 blocks of 256 threads"""
    g = torch.Generator(device="cuda").manual_seed(rows + cols)
    x = torch.randn(rows, ld, device="cuda", generator=g) * torch.exp2(torch.randint(-130, 128, (rows, ld), device="cuda",
                                                                                          generator=g).float())
    specials = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1 + 2 ** -8, 1 + 3 * 2 ** -8,
                             -(1 + 2 ** -8), 3.4e38, 2 ** -140, -(2 ** -149), 1.0], device="cuda")
    flat = x.view(-1)
    flat[:specials.numel()] = specials[:flat.numel()]
    x[:, cols:] = float("nan")   # never read
    src = Buf(rows * ld, values=x)
    out = Buf(rows * ld16, BF16)
    call("tb_f32_to_bf16", src.ptr, out.ptr, rows, cols, ld, ld16, stream())
    torch.cuda.synchronize()
    assert out.guards_intact() and src.unchanged()
    got = out.t.view(rows, ld16)
    want = x[:, :cols].cpu().to(BF16).cuda()
    nan = want.isnan()
    assert torch.equal(got[:, :cols].isnan(), nan)
    assert torch.equal(got[:, :cols].view(torch.int16)[~nan], want.view(torch.int16)[~nan])
    assert bool((got[:, cols:].view(torch.int16) == 0).all())
