"""GPU: the fp32 network building blocks in isolation against float64 - the SIMT GEMM of the fp32 backend, the AtariNet
and ResNet patch-matrix kernels, the fused policy / baseline heads and the bias-gradient column sums.

Two kinds of check:
- exact: small integers in f32 / bf16 and uint8 frames in {0, 255} (read as exactly 0.0 and 1.0) keep every product and
  partial sum below 2^24, so the kernels must equal the float64 reference bit for bit whatever their summation order or
  split count; that catches any lost, doubled or misplaced element;
- bounded: randn / random uint8 data against a bound derived from the length of each accumulation chain, and each such
  test also shows that the bound rejects the reference with one k term dropped.
Outputs and every scratch / split-K partial buffer are filled with NaN before a call, outputs carry sentinel columns
past N that must stay untouched, and a second call must give the same bits.  Data movement (patch matrices, permutes,
maxpool values and argmax taps, ReLU) is compared bit for bit with torch's unfold / max_pool2d / permutes.

Last, the heads backward at the batch sizes that used to fail: a launch past grid.y's 65535 rows (T1 * B = 65610) and a
weight-gradient scratch that grew with N (multi-task A = 18, V = 57 at T1 * B = 13770)."""
import math

import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu

NUM_SMS = 132
U32 = 2.0 ** -24
NAN = float("nan")


def lib():
    from torchbeast_b200 import _lib
    return _lib.lib()


def P(t):
    from torchbeast_b200 import _lib
    return _lib.ptr(t)


def stream():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    rc = getattr(lib(), name)(*args)
    assert rc == 0, "%s: %s" % (name, lib().tb_last_error().decode())


def rejects(name, *args):
    rc = getattr(lib(), name)(*args)
    assert rc != 0, "%s accepted a call it must reject" % name
    return lib().tb_last_error().decode()


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def ints(shape, lo, hi, g, dtype=torch.float32):
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).to(dtype)


def frames01(shape, g):
    """uint8 frames of 0 and 255 only: read as x / 255 they are exactly 0.0 and 1.0"""
    return (torch.randint(0, 2, shape, device="cuda", generator=g) * 255).to(torch.uint8)


def mm64(a, b, fa=None, fb=None, rows=1 << 16, chunk=1 << 17):
    """float64 fa(a) @ fb(b), converting blocks of rows and of the reduction dimension at a time (the conv1 products have
    10^6 rows or reduce over them)"""
    out = torch.zeros(a.shape[0], b.shape[1], dtype=torch.float64, device="cuda")
    for m0 in range(0, a.shape[0], rows):
        for k0 in range(0, a.shape[1], chunk):
            x, y = a[m0:m0 + rows, k0:k0 + chunk].double(), b[k0:k0 + chunk].double()
            out[m0:m0 + rows] += (fa(x) if fa else x) @ (fb(y) if fb else y)
    return out


def bound(K, sq, ref):
    """fp32 accumulation of K products against the float64 sum: each addition rounds by at most 2^-24 of the running sum,
    whose spread grows like sqrt(k) * rms(product), so the error's spread is about 2^-24 * sqrt(K / 2) * sqrt(sum of
    squared products) = sq.  Six times sqrt(K) * sq, plus 2^-22 |ref| for the operand (x / 255) and epilogue roundings."""
    return 6.0 * U32 * math.sqrt(K) * sq + 4.0 * U32 * ref.abs() + 1e-30


# ---------------------------------------------------------------------------------------------------------------------
# fp32 SIMT GEMM
# ---------------------------------------------------------------------------------------------------------------------
SPLITK_FLOATS = 8 << 20


def simt_splits(M, N, K, scratch=SPLITK_FLOATS, cap=128):
    """simt_splits (gemm_simt.cuh): about two waves of CTA tiles, at least four K tiles of 16 per split, the partials
    within the scratch, at most `cap`."""
    bm, bn = (128, 32) if N <= 32 else ((64 if M <= 64 else 128), 64)
    tiles = -(-M // bm) * -(-N // bn)
    s = min(-(-2 * NUM_SMS // tiles), -(-K // 16) // 4)
    if s * M * N > scratch:
        s = scratch // (M * N)
    return max(min(s, cap), 1)


def effective_splits(K, splits):
    return max(1, min(splits, -(-K // 16)))


class Gemm:
    """One tb_gemm_f32 call and its float64 reference.  layout: "nt" forward (A [M,K], B [N,K]), "nn" input gradient
    (B [K,N]), "tn" weight gradient (A stored [K,M], B [K,N]); a_u8 / b_u8 as the learner's conv1 operands."""

    def __init__(self, layout, M, N, K, a_u8=False, b_u8=False, lda=None, ldb=None, ldc=None, exact=True, seed=0,
                 bias=False, relu=0, mask=False, addend=False, accumulate=False, perm=(1, 1), scale=1.0, splits=1):
        g = gen(seed)
        ta, tb = layout == "tn", layout == "nt"
        ashape = (K, lda or M) if ta else (M, lda or K)
        bshape = (N, ldb or K) if tb else (K, ldb or N)

        def operand(shape, u8):
            if u8:
                return frames01(shape, g) if exact else torch.randint(0, 256, shape, device="cuda", generator=g).to(torch.uint8)
            return ints(shape, -3, 3, g) if exact else torch.randn(shape, device="cuda", generator=g)

        self.A, self.B = operand(ashape, a_u8), operand(bshape, b_u8)
        self.ldc = ldc or N
        # the operands as [M, K] and [K, N] views; fa / fb turn a float64 block of them into values (uint8: x / 255)
        self.Am = self.A[:K, :M].t() if ta else self.A[:M, :K]
        self.Bm = self.B[:N, :K].t() if tb else self.B[:K, :N]
        self.fa = (lambda t: t / 255.0) if a_u8 else None
        self.fb = (lambda t: t / 255.0) if b_u8 else None
        small = (lambda shape: ints(shape, -2, 2, g) if exact else torch.randn(shape, device="cuda", generator=g))
        self.bias = small((N,)) if bias else None
        self.mask = ints((M, N + 3), -1, 1, g) if mask else None
        self.addend = small((M, N + 5)) if addend else None
        self.C0 = small((M, self.ldc)) if accumulate else None
        self.args = dict(layout=layout, M=M, N=N, K=K, a_u8=a_u8, b_u8=b_u8, relu=relu, accumulate=accumulate,
                         perm=perm, scale=scale, splits=splits, ta=ta, tb=tb)
        self.acc = mm64(self.Am, self.Bm, self.fa, self.fb)
        self.ref = self.epilogue(self.acc)

    @property
    def via_scratch(self):
        a = self.args
        return effective_splits(a["K"], a["splits"]) > 1 or a["perm"] != (1, 1)

    def epilogue(self, acc):
        a = self.args
        M, N = a["M"], a["N"]
        if self.via_scratch:
            v = acc * a["scale"]
            if self.bias is not None:
                v = v + self.bias.double()
            if a["relu"]:
                v = v.clamp_min(0)
            pp, qq = a["perm"]
            n = torch.arange(N, device="cuda")
            out = torch.empty_like(v)
            out[:, (n % qq) * pp + n // qq] = v
            v = out
        else:
            v = acc
            if self.bias is not None:
                v = v + self.bias.double()
            if a["relu"]:
                v = v.clamp_min(0)
            if self.mask is not None:
                v = torch.where(self.mask[:, :N] > 0, v, torch.zeros_like(v))
            if self.addend is not None:
                v = v + self.addend[:, :N].double()
        if self.C0 is not None:
            v = v + self.C0[:, :N].double()
        return v

    def run(self):
        a = self.args
        M, N, K = a["M"], a["N"], a["K"]
        C = torch.full((M, self.ldc), NAN, device="cuda")
        if self.C0 is not None:
            C[:, :N] = self.C0[:, :N]
        s = effective_splits(K, a["splits"])
        scratch = torch.full((s * M * N + 64,), NAN, device="cuda") if self.via_scratch else None
        call("tb_gemm_f32", P(self.A), int(a["a_u8"]), P(self.B), int(a["b_u8"]), int(a["ta"]), int(a["tb"]), M, N, K,
             self.A.shape[1], self.B.shape[1], P(C), self.ldc, P(self.bias), a["relu"], P(self.mask),
             0 if self.mask is None else self.mask.shape[1], P(self.addend), 0 if self.addend is None else self.addend.shape[1],
             int(a["accumulate"]), a["perm"][0], a["perm"][1], a["scale"], a["splits"], P(scratch), stream())
        torch.cuda.synchronize()
        assert torch.isnan(C[:, N:]).all(), "write past column N"
        return C

    def check_exact(self):
        N = self.args["N"]
        C = self.run()
        assert torch.equal(C[:, :N].double(), self.ref), "%s: off by %s" % (self.args, (C[:, :N].double() - self.ref).abs().max())
        assert torch.equal(self.run()[:, :N], C[:, :N]), "a second call gave other bits"

    def check_bounded(self, drop_k):
        a = self.args
        assert not a["relu"] and self.mask is None
        C = self.run()
        sq = lambda t: t * t  # noqa: E731
        fa2 = (lambda t: sq(self.fa(t))) if self.fa else sq
        fb2 = (lambda t: sq(self.fb(t))) if self.fb else sq
        tol = self.output_order(bound(a["K"], mm64(self.Am, self.Bm, fa2, fb2).sqrt(), self.acc) * abs(a["scale"]))
        tol = tol + 4.0 * U32 * self.ref.abs()
        err = ((C[:, :a["N"]].double() - self.ref).abs() / tol).max().item()
        assert err <= 1.0, "%s: error %.3g of the bound" % (a, err)
        # the bound must see one lost k term
        col = self.Am[:, drop_k:drop_k + 1].double()
        row = self.Bm[drop_k:drop_k + 1].double()
        term = (self.fa(col) if self.fa else col) @ (self.fb(row) if self.fb else row)
        dropped = self.epilogue(self.acc - term)
        assert ((dropped - self.ref).abs() / tol).max().item() > 1.0, "the bound cannot see a dropped k term"
        C2 = self.run()
        assert torch.equal(C2[:, :a["N"]], C[:, :a["N"]])

    def output_order(self, t):
        """[M, N] in accumulator order -> the kernel's output order (the split-K reduce's column permutation)"""
        if not self.via_scratch:
            return t
        pp, qq = self.args["perm"]
        n = torch.arange(self.args["N"], device="cuda")
        out = torch.empty_like(t)
        out[:, (n % qq) * pp + n // qq] = t
        return out


def tb_splits(M, N, K, scratch=SPLITK_FLOATS, cap=128):
    return lib().tb_gemm_f32_splits(M, N, K, scratch, cap)


T1B = 81 * 32   # the learner step at T = 80, B = 32
CORE = 519      # AtariNet core width at A = 6: 512 + 1 + A
HP = 524        # padded_h(519) (lstm.cu): the row stride of the LSTM's masked h
M1, M2, M3 = T1B * 400, T1B * 81, T1B * 49

# the split counts the learner picks for its weight gradients at T = 80, B = 32 (a rule change shows up here first)
LEARNER_WGRAD = [
    # name, M (nout), N (kin), K (rows), perm, cap, expected splits
    ("fc_wgrad", 512, 3136, T1B, (49, 64), 128, 2),
    ("conv3_wgrad", 64, 576, M3, (9, 64), 128, 30),
    ("conv2_wgrad", 64, 512, M2, (16, 32), 128, 33),
    ("conv1_wgrad", 32, 256, M1, (1, 1), 128, 66),
    ("lstm_whh_wgrad", 4 * CORE, CORE, T1B, (1, 1), 64, 2),
    ("lstm_wih_wgrad", 4 * CORE, CORE, T1B, (1, 1), 64, 2),
]


@pytest.mark.parametrize("case", LEARNER_WGRAD, ids=[c[0] for c in LEARNER_WGRAD])
def test_learner_split_counts(case):
    _, M, N, K, _, cap, want = case
    assert simt_splits(M, N, K, cap=cap) == want
    assert tb_splits(M, N, K, SPLITK_FLOATS, cap) == want
    assert lib().tb_splitk_scratch_floats() == SPLITK_FLOATS


def test_split_rule_matches_restatement():
    for M in (1, 31, 32, 33, 63, 64, 65, 129, 512, 2076):
        for N in (1, 31, 32, 33, 63, 64, 65, 129, 576, 3136):
            for K in (1, 15, 16, 17, 64, 65, 4096, 200000):
                for cap in (64, 128):
                    assert tb_splits(M, N, K, SPLITK_FLOATS, cap) == simt_splits(M, N, K, cap=cap), (M, N, K, cap)
    assert tb_splits(64, 64, 10 ** 6, 64 * 64 * 5, 128) == 5  # the partials' scratch caps the count


# every product the learner runs at T = 80, B = 32 (ResNet: 64 frames of each section), exact on integer data
LEARNER_GEMMS = [
    ("conv1_fwd", dict(layout="nt", M=M1, N=32, K=256, a_u8=True, bias=True, relu=1)),
    ("conv2_fwd", dict(layout="nt", M=M2, N=64, K=512, bias=True, relu=1)),
    ("conv3_fwd", dict(layout="nt", M=M3, N=64, K=576, bias=True, relu=1)),
    ("fc_fwd", dict(layout="nt", M=T1B, N=512, K=3136, ldc=CORE, bias=True, relu=1)),
    ("fc_dgrad", dict(layout="nn", M=T1B, N=3136, K=512, lda=CORE, mask=True)),
    ("conv3_dgrad", dict(layout="nn", M=M3, N=576, K=64)),
    ("conv2_dgrad", dict(layout="nn", M=M2, N=512, K=64)),
    ("fc_wgrad", dict(layout="tn", M=512, N=3136, K=T1B, lda=CORE, perm=(49, 64), splits=2)),
    ("conv3_wgrad", dict(layout="tn", M=64, N=576, K=M3, perm=(9, 64), splits=30)),
    ("conv2_wgrad", dict(layout="tn", M=64, N=512, K=M2, perm=(16, 32), splits=33)),
    ("conv1_wgrad", dict(layout="tn", M=32, N=256, K=M1, b_u8=True, splits=66)),
    ("lstm_gates_fwd", dict(layout="nt", M=T1B, N=4 * CORE, K=CORE, bias=True)),
    ("lstm_whh_wgrad", dict(layout="tn", M=4 * CORE, N=CORE, K=T1B, ldb=HP)),
    ("lstm_wih_wgrad", dict(layout="tn", M=4 * CORE, N=CORE, K=T1B)),
    ("lstm_dgrad", dict(layout="nn", M=T1B, N=CORE, K=4 * CORE)),
    ("resnet_conv_fwd_addend", dict(layout="nt", M=64 * 42 * 42, N=16, K=144, bias=True, addend=True)),
    ("resnet_conv_fwd_addend_c32", dict(layout="nt", M=64 * 11 * 11, N=32, K=288, bias=True, relu=1, addend=True)),
    ("resnet_conv1_u8_fwd", dict(layout="nt", M=64 * 84 * 84, N=16, K=36, a_u8=True, lda=40, ldb=40, bias=True)),
    ("resnet_conv1_u8_wgrad", dict(layout="tn", M=16, N=36, K=64 * 84 * 84, b_u8=True, ldb=40,
                                   splits=simt_splits(16, 36, 64 * 84 * 84))),
]


@pytest.mark.parametrize("name,kw", LEARNER_GEMMS, ids=[c[0] for c in LEARNER_GEMMS])
def test_gemm_learner_shapes_exact(name, kw):
    if "lstm" in name and "wgrad" in name:
        kw = dict(kw, splits=simt_splits(kw["M"], kw["N"], kw["K"], cap=64))
    Gemm(**kw).check_exact()


EDGE = (1, 31, 32, 33, 63, 64, 65, 129)
LAYOUTS = [("nt", False, False), ("nt", True, False), ("nn", False, False), ("tn", False, False), ("tn", False, True)]


@pytest.mark.parametrize("layout,a_u8,b_u8", LAYOUTS, ids=["fwd", "fwd_u8", "dgrad", "wgrad", "wgrad_u8"])
def test_gemm_edges_exact(layout, a_u8, b_u8):
    """M, N across all three tile shapes and the reduce's 4-column vector / scalar tail; K around one K tile."""
    for M in EDGE:
        for N in EDGE:
            Gemm(layout, M, N, 17, a_u8=a_u8, b_u8=b_u8, ldc=N + 3, seed=M * 131 + N, bias=True).check_exact()
    for K in (1, 15, 16, 17):
        Gemm(layout, 33, 65, K, a_u8=a_u8, b_u8=b_u8, seed=K).check_exact()
        Gemm(layout, 65, 33, K, a_u8=a_u8, b_u8=b_u8, seed=K, splits=4, perm=(11, 3), scale=0.5).check_exact()


@pytest.mark.parametrize("M,N", [(1, 1), (33, 31), (65, 129), (129, 64), (31, 33)])
def test_gemm_splitk_edges_exact(M, N):
    """split-K partials: an empty trailing slice (5 K tiles over 4 splits: 2, 2, 1, 0), more splits than K tiles
    (clamped), every epilogue of the reduce, and the permuted un-pack."""
    perm = next(((p, N // p) for p in (3, 2, 5, 7) if N % p == 0 and N // p > 1), (1, 1))
    for K, splits in ((80, 4), (80, 3), (33, 8), (16 * 9, 5), (1000, 7)):
        for layout, a_u8, b_u8 in LAYOUTS:
            Gemm(layout, M, N, K, a_u8=a_u8, b_u8=b_u8, splits=splits, seed=K + splits, ldc=N + 2).check_exact()
        Gemm("tn", M, N, K, splits=splits, perm=perm, bias=True, relu=1, scale=0.25, accumulate=True, seed=7).check_exact()
        Gemm("tn", M, N, K, b_u8=True, splits=splits, perm=perm, scale=2.0, seed=8).check_exact()


def test_gemm_direct_epilogues_exact():
    for M, N in ((129, 65), (33, 32), (1, 1), (64, 63)):
        for layout, a_u8, b_u8 in LAYOUTS:
            Gemm(layout, M, N, 40, a_u8=a_u8, b_u8=b_u8, ldc=N + 4, bias=True, relu=1, mask=True, addend=True,
                 accumulate=True, seed=M + N).check_exact()


def test_gemm_rejects_ignored_epilogue():
    """each path applies only part of the epilogue: asking for the rest is an error, not a silently different result"""
    g = Gemm("tn", 64, 64, 256, splits=4, mask=True)
    C = torch.zeros(64, 64, device="cuda")
    scratch = torch.zeros(4 * 64 * 64, device="cuda")
    base = [P(g.A), 0, P(g.B), 0, 1, 0, 64, 64, 256, 64, 64, P(C), 64, None, 0]
    err = rejects("tb_gemm_f32", *base, P(g.mask), g.mask.shape[1], None, 0, 0, 1, 1, 1.0, 4, P(scratch), stream())
    assert "mask" in err
    err = rejects("tb_gemm_f32", *base, None, 0, P(g.mask), g.mask.shape[1], 0, 8, 8, 1.0, 1, P(scratch), stream())
    assert "addend" in err
    err = rejects("tb_gemm_f32", *base, None, 0, None, 0, 0, 1, 1, 0.5, 1, P(scratch), stream())
    assert "scale" in err
    # K = 16 is one K tile: splits clamp to 1, so the direct path (with its mask) is taken and the call is valid
    call("tb_gemm_f32", *base[:8], 16, *base[9:], P(g.mask), g.mask.shape[1], None, 0, 0, 1, 1, 1.0, 4, P(scratch), stream())
    err = rejects("tb_gemm_f32", P(g.A), 1, P(g.B), 1, 1, 0, 64, 64, 256, 64, 64, P(C), 64, None, 0, None, 0, None, 0, 0, 1, 1,
                  1.0, 1, None, stream())
    assert "no kernel" in err
    torch.cuda.synchronize()


BOUNDED = [
    ("fc_fwd", dict(layout="nt", M=T1B, N=512, K=3136, ldc=CORE, bias=True), 3135),
    ("conv1_fwd_u8", dict(layout="nt", M=4096, N=32, K=256, a_u8=True, bias=True), 100),
    ("fc_dgrad", dict(layout="nn", M=T1B, N=3136, K=512, lda=CORE), 511),
    ("conv3_wgrad_split", dict(layout="tn", M=64, N=576, K=M3, perm=(9, 64), splits=30), M3 - 1),
    ("conv1_wgrad_u8_split", dict(layout="tn", M=32, N=256, K=M1, b_u8=True, splits=66), 12345),
    ("lstm_wgrad", dict(layout="tn", M=4 * CORE, N=CORE, K=T1B, ldb=HP, splits=2), 0),
    ("edge_split_tail", dict(layout="tn", M=65, N=33, K=80, splits=4, perm=(11, 3), scale=0.5), 79),
]


@pytest.mark.parametrize("name,kw,drop_k", BOUNDED, ids=[c[0] for c in BOUNDED])
def test_gemm_bounded_random(name, kw, drop_k):
    Gemm(exact=False, seed=3, **kw).check_bounded(drop_k)


# ---------------------------------------------------------------------------------------------------------------------
# AtariNet patch matrices and pointwise kernels
# ---------------------------------------------------------------------------------------------------------------------
def unfold_rows(x_nchw, KH, KW, S, padding=0):
    """[N,C,H,W] -> [N*OH*OW, C*KH*KW] with k = (c*KH + kh)*KW + kw (torch's unfold order)"""
    N = x_nchw.shape[0]
    u = Fn.unfold(x_nchw, (KH, KW), stride=S, padding=padding)  # [N, C*KH*KW, L]
    return u.transpose(1, 2).reshape(-1, u.shape[1])


@pytest.mark.parametrize("N,C,H,W,KH,KW,S", [(3, 4, 84, 84, 8, 8, 4), (2, 4, 84, 84, 8, 8, 4), (2, 3, 21, 22, 5, 3, 2),
                                             (1, 1, 9, 9, 8, 8, 1), (2, 4, 86, 86, 8, 8, 4)])
def test_im2col_u8_nchw(N, C, H, W, KH, KW, S):
    g = gen(11)
    fr = torch.randint(0, 256, (N, C, H, W), device="cuda", generator=g).to(torch.uint8)
    OH, OW = (H - KH) // S + 1, (W - KW) // S + 1
    col = torch.full((N * OH * OW * C * KH * KW + 8,), 77, dtype=torch.uint8, device="cuda")
    call("tb_im2col_u8_nchw", P(fr), P(col), N, C, H, W, KH, KW, S, stream())
    ref = unfold_rows(fr.float(), KH, KW, S).to(torch.uint8).reshape(-1)
    assert torch.equal(col[:-8], ref)
    assert (col[-8:] == 77).all()


def nhwc_unfold(act, KH, KW, S):
    """NHWC [N,H,W,C] -> [N*OH*OW, KH*KW*C] with k = (kh*KW + kw)*C + c"""
    N, H, W, C = act.shape
    u = Fn.unfold(act.permute(0, 3, 1, 2), (KH, KW), stride=S)  # [N, C*KH*KW, L]
    L = u.shape[2]
    return u.reshape(N, C, KH * KW, L).permute(0, 3, 2, 1).reshape(N * L, KH * KW * C)


@pytest.mark.parametrize("N,H,W,C,KH,KW,S", [(3, 20, 20, 32, 4, 4, 2), (3, 9, 9, 64, 3, 3, 1), (2, 7, 10, 4, 3, 2, 3)])
def test_im2col_col2im_f32_nhwc(N, H, W, C, KH, KW, S):
    g = gen(12)
    act = torch.randn(N, H, W, C, device="cuda", generator=g)
    OH, OW = (H - KH) // S + 1, (W - KW) // S + 1
    K = KH * KW * C
    col = torch.full((N * OH * OW, K), NAN, device="cuda")
    call("tb_im2col_f32_nhwc", P(act), P(col), N, H, W, C, KH, KW, S, stream())
    assert torch.equal(col, nhwc_unfold(act, KH, KW, S))
    # col2im: the adjoint of the above on integer data (exact), with and without the ReLU mask of the forward activation
    dcol = ints((N * OH * OW, K), -4, 4, g)
    dcol_nchw = dcol.double().reshape(N, OH * OW, KH * KW, C).permute(0, 3, 2, 1).reshape(N, C * KH * KW, OH * OW)
    ref = Fn.fold(dcol_nchw, (H, W), (KH, KW), stride=S).permute(0, 2, 3, 1)
    for mask in (None, act):
        dact = torch.full((N, H, W, C), NAN, device="cuda")
        call("tb_col2im_f32_nhwc", P(dcol), P(mask), P(dact), N, H, W, C, KH, KW, S, stream())
        want = ref if mask is None else torch.where(act > 0, ref, torch.zeros_like(ref))
        assert torch.equal(dact.double(), want)


def test_permute_relu_mask_core_extras():
    g = gen(13)
    for O, Pp, Q in ((64, 16, 32), (512, 49, 64), (3, 1, 7), (5, 7, 1)):
        x = torch.randn(O, Pp * Q, device="cuda", generator=g)
        out = torch.full_like(x, NAN)
        call("tb_permute_pq", P(x), P(out), O, Pp, Q, stream())
        assert torch.equal(out, x.reshape(O, Q, Pp).transpose(1, 2).reshape(O, Pp * Q))
    # ReLU mask in place on a strided view: columns >= ncols untouched, zero exactly where !(Y > 0) (NaN included)
    M, nc, ldx, ldy = 2592, 512, CORE, CORE + 2
    X = torch.randn(M, ldx, device="cuda", generator=g)
    Y = torch.randn(M, ldy, device="cuda", generator=g)
    Y[0, :4] = torch.tensor([0.0, -0.0, NAN, 1e-30])
    X0 = X.clone()
    call("tb_relu_mask_f32", P(X), P(Y), M, nc, ldx, ldy, stream())
    want = X0.clone()
    want[:, :nc] = torch.where(Y[:, :nc] > 0, X0[:, :nc], torch.zeros_like(X0[:, :nc]))
    assert torch.equal(X, want)
    # core extras: clipped reward and the last-action one-hot behind the first F columns, nothing else written
    for A in (6, 18, 0):
        N, F = 2592, 512
        ld = F + 1 + A + 2
        core = torch.full((N, ld), NAN, device="cuda")
        reward = torch.randn(N, device="cuda", generator=g) * 3
        reward[:4] = torch.tensor([1.0, -1.0, 1.0000001, -7.0])
        last = torch.randint(0, max(A, 1), (N,), device="cuda", generator=g)
        call("tb_core_extras", P(core), ld, N, F, P(reward), P(last) if A else None, A, stream())
        assert torch.equal(core[:, F], reward.clamp(-1, 1))
        if A:
            assert torch.equal(core[:, F + 1:F + 1 + A], Fn.one_hot(last, A).float())
        assert torch.isnan(core[:, :F]).all() and torch.isnan(core[:, F + 1 + A:]).all()


# ---------------------------------------------------------------------------------------------------------------------
# ResNet patch-matrix path (f32 and bf16)
# ---------------------------------------------------------------------------------------------------------------------
DT = {0: torch.float32, 1: torch.bfloat16}


@pytest.mark.parametrize("dtype", [0, 1], ids=["f32", "bf16"])
@pytest.mark.parametrize("N,H,W,C", [(4, 42, 42, 16), (3, 11, 11, 32), (2, 5, 7, 8), (1, 1, 1, 16)])
def test_im2col3x3_col2im3x3(dtype, N, H, W, C):
    g = gen(21)
    dt = DT[dtype]
    x = ints((N, H, W, C), -3, 3, g, dt) if dtype else torch.randn(N, H, W, C, device="cuda", generator=g)
    ldk = 9 * C + (8 if dtype else 4)
    for relu_in in (0, 1):
        col = torch.full((N * H * W, ldk), NAN, dtype=dt, device="cuda")
        call("tb_im2col3x3", P(x), P(col), N, H, W, C, ldk, relu_in, dtype, stream())
        src = x.float().clamp_min(0) if relu_in else x.float()
        u = Fn.unfold(src.permute(0, 3, 1, 2), 3, padding=1).reshape(N, C, 9, H * W).permute(0, 3, 2, 1)
        assert torch.equal(col[:, :9 * C].float(), u.reshape(N * H * W, 9 * C))
    # col2im3x3 (gather form) on integer data, with the ReLU mask and the residual addend each on and off
    dcol = ints((N * H * W, ldk), -3, 3, g, dt)
    dcol[:, 9 * C:] = NAN  # the k padding must not be read
    d = dcol[:, :9 * C].double().reshape(N, H * W, 9, C).permute(0, 3, 2, 1).reshape(N, 9 * C, H * W)
    ref = Fn.fold(d, (H, W), 3, padding=1).permute(0, 2, 3, 1)
    addend = ints((N, H, W, C), -5, 5, g, dt)
    for relu_src in (None, x):
        for add in (None, addend):
            dx = torch.full((N, H, W, C), NAN, dtype=dt, device="cuda")
            call("tb_col2im3x3", P(dcol), P(relu_src), P(add), P(dx), N, H, W, C, ldk, dtype, stream())
            want = ref if relu_src is None else torch.where(x > 0, ref, torch.zeros_like(ref))
            want = want if add is None else want + add.double()
            assert torch.equal(dx.double(), want)


@pytest.mark.parametrize("dtype", [0, 1], ids=["u8", "bf16"])
@pytest.mark.parametrize("N,C,H,W,ldk", [(3, 4, 84, 84, 40), (2, 3, 64, 64, 32), (2, 1, 9, 7, 16), (2, 16, 12, 10, 144),
                                         (2, 5, 8, 8, 48), (1, 3, 72, 96, 27)])
def test_im2col3x3_u8(dtype, N, C, H, W, ldk):
    """both kernels: up to 4 channels (whole patch row in registers, 16-byte stores at ldk = 40) and the wide one"""
    g = gen(22)
    fr = torch.randint(0, 256, (N, C, H, W), device="cuda", generator=g).to(torch.uint8)
    out_dt = torch.bfloat16 if dtype else torch.uint8
    col = torch.full((N * H * W, ldk), 99, dtype=out_dt, device="cuda")
    call("tb_im2col3x3_u8", P(fr), P(col), N, C, H, W, ldk, dtype, stream())
    ref = unfold_rows(fr.float(), 3, 3, 1, padding=1)
    assert torch.equal(col[:, :9 * C].float(), ref)
    assert (col[:, 9 * C:].float() == 0).all(), "the k padding is zeroed"


def torch_pool(x):
    """float64 nn.MaxPool2d(3, 2, 1) on NHWC (CPU: first maximum wins) -> y, the argmax tap kh*3 + kw"""
    N, H, W, C = x.shape
    y, idx = Fn.max_pool2d(x.double().cpu().permute(0, 3, 1, 2), 3, 2, 1, return_indices=True)
    OH, OW = y.shape[2], y.shape[3]
    oy = torch.arange(OH).view(1, 1, OH, 1)
    ox = torch.arange(OW).view(1, 1, 1, OW)
    tap = (idx // W - (2 * oy - 1)) * 3 + (idx % W - (2 * ox - 1))
    return y.permute(0, 2, 3, 1).cuda(), tap.permute(0, 2, 3, 1).to(torch.uint8).cuda()


@pytest.mark.parametrize("dtype", [0, 1], ids=["f32", "bf16"])
@pytest.mark.parametrize("N,H,W,C", [(4, 84, 84, 16), (3, 42, 42, 32), (2, 21, 21, 32), (2, 8, 9, 16), (1, 1, 2, 8)])
def test_maxpool3x3s2(dtype, N, H, W, C):
    g = gen(23)
    dt = DT[dtype]
    for tied in (False, True):
        x = ints((N, H, W, C), 0, 2, g, dt) if tied else torch.randn(N, H, W, C, device="cuda", generator=g).to(dt)
        OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.full((N, OH, OW, C), NAN, dtype=dt, device="cuda")
        arg = torch.full((N, OH, OW, C), 200, dtype=torch.uint8, device="cuda")
        call("tb_maxpool3x3s2_fwd", P(x), P(y), P(arg), N, H, W, C, dtype, stream())
        yref, tap = torch_pool(x)
        assert torch.equal(y.double(), yref)
        assert torch.equal(arg, tap)
        if dtype == 0:  # the f32 entry the shifted-window path uses is the same kernel
            y2, arg2 = torch.empty_like(y), torch.empty_like(arg)
            call("tb_maxpool3x3s2_fwd_f32", P(x), P(y2), P(arg2), N, H, W, C, stream())
            assert torch.equal(y2, y) and torch.equal(arg2, arg)
        # backward against float64 autograd of max_pool2d (same tie rule), integer cotangents: exact in bf16 as well
        dy = ints((N, OH, OW, C), -4, 4, g, dt)
        dx = torch.full((N, H, W, C), NAN, dtype=dt, device="cuda")
        call("tb_maxpool3x3s2_bwd", P(arg), P(dy), P(dx), N, H, W, C, dtype, stream())
        xd = x.double().cpu().permute(0, 3, 1, 2).requires_grad_()
        Fn.max_pool2d(xd, 3, 2, 1).backward(dy.double().cpu().permute(0, 3, 1, 2))
        assert torch.equal(dx.double().cpu(), xd.grad.permute(0, 2, 3, 1))


@pytest.mark.parametrize("dtype", [0, 1], ids=["f32", "bf16"])
def test_relu_fwd_bwd(dtype):
    g = gen(24)
    dt = DT[dtype]
    n = 2592 * 256 + 8 * 37
    x = torch.randn(n, device="cuda", generator=g).to(dt)
    x[:6] = torch.tensor([0.0, -0.0, NAN, float("inf"), -float("inf"), 1e-30]).to(dt)
    dy = torch.randn(n, device="cuda", generator=g).to(dt)
    y, dx = torch.full_like(x, NAN), torch.full_like(x, NAN)
    call("tb_relu_fwd", P(x), P(y), n, dtype, stream())
    call("tb_relu_bwd", P(x), P(dy), P(dx), n, dtype, stream())
    torch.cuda.synchronize()
    assert torch.equal(y[6:], torch.relu(x[6:])) and torch.equal(y[:2].float(), torch.zeros(2, device="cuda"))
    assert torch.equal(y[3:6].float(), torch.tensor([float("inf"), 0.0, 1e-30], device="cuda").to(dt).float())
    assert torch.equal(dx, torch.where(x > 0, dy, torch.zeros_like(dy)))
    assert "dtype" in rejects("tb_relu_fwd", P(x), P(y), n, 2, stream())


# ---------------------------------------------------------------------------------------------------------------------
# bias-gradient column sums
# ---------------------------------------------------------------------------------------------------------------------
COLSUM_M = [1, 7, 63, 64, 65, 4095, 4096, 16387, 256 * 64 + 1, M1]


def colsum_call(X, M, ncols, ld, bf16, lo_off=0):
    scratch = torch.full((lib().tb_colsum_scratch_floats(max(ncols, 512)),), NAN, device="cuda")
    out = torch.full((ncols + 3,), NAN, device="cuda")
    if bf16:
        call("tb_colsum_bf16", P(X), P(out), M, ncols, ld, P(scratch), lo_off, stream())
    else:
        call("tb_colsum_f32", P(X), P(out), M, ncols, ld, P(scratch), stream())
    torch.cuda.synchronize()
    assert torch.isnan(out[ncols:]).all()
    return out[:ncols]


@pytest.mark.parametrize("M", COLSUM_M)
def test_colsum_exact(M):
    g = gen(31)
    cases = [(32, 32), (64, 64), (8, 8), (16, 16), (33, 33), (512, CORE), (2076, 2076)] if M <= 4 * T1B else \
        [(32, 32), (64, 64)]
    for ncols, ld in cases:
        if M * ld > 40e6:
            continue
        X = ints((M, ld), -4, 4, g)
        ref = X[:, :ncols].double().sum(0)
        out = colsum_call(X, M, ncols, ld, False)
        assert torch.equal(out.double(), ref), (M, ncols, ld)
        assert torch.equal(colsum_call(X, M, ncols, ld, False), out)
        # bf16: the dense 16-byte path (ld == ncols in {8,16,32,64}, M >= 4096) and the strided one, with and without a
        # lo plane (the split-bf16 gradient's second plane) behind the hi plane
        for ldb in (ld, ld + 8):
            for lo in (False, True):
                Xb = torch.full((2 if lo else 1, M, ldb), NAN, dtype=torch.bfloat16, device="cuda")
                Xb[0, :, :ncols] = ints((M, ncols), -4, 4, g, torch.bfloat16)
                want = Xb[0, :, :ncols].double().sum(0)
                if lo:
                    Xb[1, :, :ncols] = ints((M, ncols), -1, 1, g, torch.bfloat16)
                    want = want + Xb[1, :, :ncols].double().sum(0)
                out = colsum_call(Xb, M, ncols, ldb, True, M * ldb if lo else 0)
                assert torch.equal(out.double(), want), (M, ncols, ldb, lo)


def test_colsum_bounded_random():
    """randn at the conv1 bias gradient's 10^6 rows: a two-stage fp32 sum, bound by the chain length; the bound sees one
    lost row"""
    g = gen(32)
    for M, ncols, ld in ((M1, 32, 32), (M2, 64, 64), (T1B, 512, CORE), (100, 33, 40)):
        X = torch.randn(M, ld, device="cuda", generator=g)
        ref = X[:, :ncols].double().sum(0)
        sq = X[:, :ncols].double().pow(2).sum(0).sqrt()
        tol = bound(M, sq, ref)
        out = colsum_call(X, M, ncols, ld, False)
        assert ((out.double() - ref).abs() / tol).max() <= 1.0
        r = X[:, :ncols].abs().argmax(0)
        dropped = ref - X[r, torch.arange(ncols, device="cuda")].double()
        assert ((dropped - ref).abs() / tol).max() > 1.0
        Xb = X.to(torch.bfloat16)
        refb = Xb[:, :ncols].double().sum(0)
        outb = colsum_call(Xb, M, ncols, ld, True)
        assert ((outb.double() - refb).abs() / bound(M, Xb[:, :ncols].double().pow(2).sum(0).sqrt(), refb)).max() <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# fused policy / baseline heads
# ---------------------------------------------------------------------------------------------------------------------
HEADS_AVF = [(1, 1, 1), (6, 1, 519), (18, 1, 531), (31, 64, 519), (18, 57, 531), (6, 4, 257), (1, 1, 12288)]
HEADS_N = [1, 63, 64, 65, 2592, 65610]


def heads_run(x, ldx, Wp, bp, Wb, bb, dl, db, N, F, A, V, lddx):
    logits = torch.full((N, A), NAN, device="cuda")
    base = torch.full((N, V), NAN, device="cuda")
    call("tb_heads_forward", P(x), ldx, P(Wp), P(bp), P(Wb), P(bb), N, F, A, V, P(logits), P(base), stream())
    dx = torch.full((N, lddx), NAN, device="cuda")
    g = [torch.full_like(t, NAN) for t in (Wp, bp, Wb, bb)]
    scratch = torch.full((lib().tb_heads_scratch_floats(N, F, A, V),), NAN, device="cuda")
    call("tb_heads_backward", P(x), ldx, P(Wp), P(Wb), P(dl), P(db), N, F, A, V, P(dx), lddx, *[P(t) for t in g], P(scratch),
         stream())
    torch.cuda.synchronize()
    assert torch.isnan(dx[:, F:]).all(), "dx written past column F"
    return logits, base, dx, g


def heads_inputs(N, F, A, V, ldx, exact, seed):
    g = gen(seed)
    mk = (lambda s: ints(s, -2, 2, g)) if exact else (lambda s: torch.randn(s, device="cuda", generator=g))
    x = torch.full((N, ldx), NAN, device="cuda")  # columns past F must not be read
    x[:, :F] = mk((N, F))
    return x, mk((A, F)), mk((A,)), mk((V, F)), mk((V,)), mk((N, A)), mk((N, V))


def heads_ref(x, Wp, bp, Wb, bb, dl, db, F):
    x = x[:, :F].double()
    d = lambda t: t.double()  # noqa: E731
    return (x @ d(Wp).t() + d(bp), x @ d(Wb).t() + d(bb), d(dl) @ d(Wp) + d(db) @ d(Wb),
            [d(dl).t() @ x, d(dl).sum(0), d(db).t() @ x, d(db).sum(0)])


@pytest.mark.parametrize("A,V,F", HEADS_AVF, ids=["%d-%d-%d" % c for c in HEADS_AVF])
def test_heads_exact(A, V, F):
    for N in HEADS_N:
        if N * F > 4e7:
            continue
        for ldx, lddx in ((F, F), (F + 5, F + 3)) if N in (65, 2592) else ((F, F),):
            inp = heads_inputs(N, F, A, V, ldx, True, N + F)
            logits, base, dx, g = heads_run(inp[0], ldx, *inp[1:], N, F, A, V, lddx)
            rl, rb, rdx, rg = heads_ref(*inp, F)
            assert torch.equal(logits.double(), rl), (A, V, F, N)
            assert torch.equal(base.double(), rb), (A, V, F, N)
            assert torch.equal(dx[:, :F].double(), rdx), (A, V, F, N)
            for got, want, name in zip(g, rg, ("dWp", "dbp", "dWb", "dbb")):
                assert torch.equal(got.double(), want), (name, A, V, F, N)
            again = heads_run(inp[0], ldx, *inp[1:], N, F, A, V, lddx)
            assert torch.equal(again[0], logits) and torch.equal(again[1], base)
            assert torch.equal(again[2][:, :F], dx[:, :F]) and all(torch.equal(a, b) for a, b in zip(again[3], g))


def test_heads_bounded_random():
    """randn at the learner's shapes: the forward's F-long and the weight gradient's N-long fp32 chains, bound by their
    length; each bound sees one dropped term"""
    for N, A, V, F in ((2592, 6, 1, 519), (65610, 18, 57, 531), (1000, 1, 1, 12288)):
        inp = heads_inputs(N, F, A, V, F, False, 5)
        x, Wp, bp, Wb, bb, dl, db = inp
        logits, base, dx, g = heads_run(x, F, Wp, bp, Wb, bb, dl, db, N, F, A, V, F)
        rl, rb, rdx, rg = heads_ref(*inp, F)
        x64 = x.double()
        sq_l = ((x64 ** 2) @ (Wp.double() ** 2).t()).sqrt()
        tol = bound(F, sq_l, rl)
        assert ((logits.double() - rl).abs() / tol).max() <= 1.0
        drop = rl - x64[:, -1:] * Wp.double()[:, -1]
        assert ((drop - rl).abs() / tol).max() > 1.0
        sq_w = ((dl.double() ** 2).t() @ (x64 ** 2)).sqrt()
        tol = bound(N, sq_w, rg[0])
        assert ((g[0].double() - rg[0]).abs() / tol).max() <= 1.0
        drop = rg[0] - dl.double()[N // 2:N // 2 + 1].t() @ x64[N // 2:N // 2 + 1]
        assert ((drop - rg[0]).abs() / tol).max() > 1.0
        tol = bound(A + V, ((dl.double() ** 2) @ (Wp.double() ** 2) + (db.double() ** 2) @ (Wb.double() ** 2)).sqrt(), rdx)
        assert ((dx.double() - rdx).abs() / tol).max() <= 1.0
        tol = bound(N, db.double().pow(2).sum(0).sqrt(), rg[3])
        assert ((g[3].double() - rg[3]).abs() / tol).max() <= 1.0
        tol = bound(F, ((x64 ** 2) @ (Wb.double() ** 2).t()).sqrt(), rb)
        assert ((base.double() - rb).abs() / tol).max() <= 1.0


def heads_slabs(N):
    """heads.cu: 64-row slabs while that takes at most 120 of them, else the fewest rows per slab that keep it at 120"""
    rows = 64 if -(-N // 64) <= 120 else -(-N // 120)
    return -(-N // rows)


def test_heads_sizes():
    h = lib()
    # the weight-gradient scratch stops growing with N: at most 120 slabs of (A + V) x (F + 1) partials
    for N in (1, 63, 64, 65, 2592, 64 * 120, 64 * 120 + 1, 13770, 65610, 10 ** 7):
        assert h.tb_heads_scratch_floats(N, 531, 18, 57) == heads_slabs(N) * 75 * 532 <= 120 * 75 * 532
    assert heads_slabs(2592) == 41 and heads_slabs(64 * 120) == 120 and heads_slabs(65610) == 120
    assert h.tb_heads_scratch_floats(10 ** 7, 700, 31, 64) == 120 * 95 * 701 <= 8 << 20
    x = torch.zeros(4, 12289, device="cuda")
    w = torch.zeros(64 * 12289, device="cuda")
    out = torch.zeros(4 * 64, device="cuda")
    assert "bad sizes" in rejects("tb_heads_forward", P(x), 12289, P(w), P(w), P(w), P(w), 4, 12289, 1, 1, P(out), P(out),
                                  stream())
    assert "bad sizes" in rejects("tb_heads_forward", P(x), 12288, P(w), P(w), P(w), P(w), 4, 12288, 32, 1, P(out), P(out),
                                  stream())
    assert "bad sizes" in rejects("tb_heads_forward", P(x), 12288, P(w), P(w), P(w), P(w), 4, 12288, 1, 65, P(out), P(out),
                                  stream())


# ---------------------------------------------------------------------------------------------------------------------
# the AtariNet backward at the batch sizes the heads used to refuse
# ---------------------------------------------------------------------------------------------------------------------
def atarinet_bias_grads(T1, B, A, V, precision):
    """tb_atarinet_backward on integer-valued cotangents: the policy / baseline bias gradients must be their float64
    column sums exactly.  They do not depend on the activations, so no forward is needed (the workspace is zeroed)."""
    h = lib()
    N = T1 * B
    core = 512 + 1 + A
    nparam = h.tb_atarinet_param_count(A, V, 0)
    wsb = h.tb_atarinet_workspace_bytes(T1, B, A, 0, precision)
    need = wsb + 4 * (2 * nparam + N * (A + V)) + (256 << 20)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("the GPU is shared: %.1f GB free, this backward needs %.1f GB" % (free / 2 ** 30, need / 2 ** 30))
    g = gen(41)
    params = torch.randn(nparam, device="cuda", generator=g) * 0.01
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    dl = ints((T1, B, A), -4, 4, g)
    db = ints((T1, B, V), -4, 4, g)
    grads = torch.full((nparam,), NAN, device="cuda")
    call("tb_atarinet_backward", P(dl), P(db), None, P(params), T1, B, A, V, 0, precision, P(ws), P(grads), 3, stream())
    torch.cuda.synchronize()
    bb = grads[nparam - V:]
    bp = grads[nparam - V - V * core - A:nparam - V - V * core]
    assert torch.equal(bp.double(), dl.double().reshape(N, A).sum(0))
    assert torch.equal(bb.double(), db.double().reshape(N, V).sum(0))
    # core_out is zero in the zeroed workspace, so the heads' weight gradients are exact zeros
    assert (grads[nparam - V - V * core - A - A * core:nparam - V - V * core - A] == 0).all()
    assert (grads[nparam - V - V * core:nparam - V] == 0).all()


def test_atarinet_backward_heads_scratch_at_13770_rows():
    """A = 18, V = 57 at T1 * B = 13770: the heads' weight-gradient partials used to outgrow the split-K scratch
    ("heads scratch too small" from N > 13440)"""
    atarinet_bias_grads(81, 170, 18, 57, 2)


def test_atarinet_backward_heads_past_65535_rows():
    """T1 * B = 65610 >= 65536: the heads' input-gradient kernel put the rows on grid.y and failed to launch"""
    atarinet_bias_grads(81, 810, 6, 1, 2)
