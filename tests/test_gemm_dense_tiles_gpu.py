"""GPU: the split-bf16 dense GEMM (gemm_tc_kernel) at every tile width its launch code chooses per call.

Each case below makes gemm_block_n pick the BLOCK_N given with it (restated in `block_n`, checked first so that a
change of the rule shows up here rather than as a silently lost case).  Products are checked against float64 torch on the
hi + lo operand values within tests/sw_image.py's tolerance, and the reference without the lo(A) . hi(B) product must lie
at least ten times outside it, so the bound also tells whether the lo planes took part.  Tile widths must not change any sum: rows computed inside a 2592-row call
are compared bit for bit with the same rows computed by a short call that picks another width.  Last, the standalone
split-bf16 LSTM at AtariNet's shape (B = 32, H = 519, 81 steps: its projections and weight gradients are the 2592-row
GEMMs of the learner step) against float64 torch.nn.LSTM."""
import ctypes
from collections import namedtuple

import numpy as np
import pytest
import torch

from tests import sw_image as S

pytestmark = pytest.mark.gpu

NUM_SMS = 132


def block_n(M, N, splits, b_mn):
    """gemm_block_n (gemm_tc.cu): fewest waves x issued columns on the busiest CTA, ties to the wider tile."""
    if not b_mn and N <= 32:
        return 32
    tiles_m = -(-M // 128)
    cost = {bn: -(-(tiles_m * -(-N // bn) * splits) // NUM_SMS) * bn for bn in (128, 64)}
    return 128 if cost[128] <= cost[64] else 64


def planes(x, ld):
    """fp32 [rows, cols] -> bf16 [2, rows, ld] (hi plane, lo plane, zero columns past cols), lo offset, fp64 hi, fp64 lo."""
    rows, cols = x.shape
    buf = torch.zeros(2, rows, ld, dtype=torch.bfloat16, device="cuda")
    hi, lo = S.split(x)
    buf[0, :, :cols], buf[1, :, :cols] = hi, lo
    return buf, rows * ld, hi.double(), lo.double()


# float64 result, the same without the lo(A) . hi(B) product, the RMS product size and the bias (sw_image.tolerance)
Ref = namedtuple("Ref", "value dropped_lo scale extra")


def rup8(n):
    return (n + 7) // 8 * 8


def gemm(M, N, K, layout, splits, epi, seed=0, gen_m=None):
    """One tb_gemm_bf16x3_ex call; returns C, the bf16 hi / lo outputs (EPI 1 / 2 without split-K) and the float64
    reference.  layout: "kk" forward (A [M,K], B [N,K]), "km" input gradient (B stored [K,N]), "mm" weight gradient
    (A stored [K,M], B [K,N]).  epi: 0 plain store, 1 scale / bias / ReLU, 2 + bf16 ReLU mask.  gen_m: draw the
    M-indexed inputs for gen_m rows and use the first M, so that calls of different M see the same leading rows."""
    from torchbeast_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(seed)
    a_mn, b_mn = layout == "mm", layout != "kk"
    gm = gen_m or M
    Ax = torch.randn((K, gm) if a_mn else (gm, K), device="cuda", generator=g)
    Ax = (Ax[:, :M] if a_mn else Ax[:M]).contiguous()
    Bx = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g)
    lda, ldb = rup8(Ax.shape[1]), rup8(Bx.shape[1])
    Ab, a_lo, Ah, Al = planes(Ax, lda)
    Bb, b_lo, Bh, Bl = planes(Bx, ldb)
    mat = lambda a, b: (a.t() if a_mn else a) @ (b if b_mn else b.t())
    acc, acc_drop = mat(Ah + Al, Bh + Bl), mat(Ah, Bh + Bl) + mat(Al, Bl)
    scale, bias, relu, mask = 1.0, None, 0, None
    if epi >= 1:
        scale, relu = 0.75, 1
        bias = torch.randn(N, device="cuda", generator=g)
    if epi == 2:
        mask = torch.zeros(M, rup8(N), dtype=torch.bfloat16, device="cuda")
        mask[:, :N] = torch.randn(gm, N, device="cuda", generator=g)[:M].to(torch.bfloat16)

    def epilogue(x):
        if epi >= 1:
            x = torch.relu(x * scale + bias.double())
        return torch.where(mask[:, :N].double() > 0, x, torch.zeros_like(x)) if epi == 2 else x
    ref = Ref(epilogue(acc), epilogue(acc_drop), S.rms(Ah + Al) * S.rms(Bh + Bl) * scale,
              bias.double() if bias is not None else None)
    C = torch.full((M, N), float("nan"), device="cuda")
    C16 = torch.zeros(2, M, rup8(N), dtype=torch.bfloat16, device="cuda") if epi >= 1 and splits == 1 else None
    part = torch.empty(splits * M * ((N + 31) // 32 * 32), device="cuda") if splits > 1 else None
    p = _lib.ptr
    rc = _lib.lib().tb_gemm_bf16x3_ex(p(Ab), p(Bb), M, N, K, lda, ldb, int(a_mn), int(b_mn), a_lo, b_lo, p(C), N, p(C16),
                                      rup8(N), M * rup8(N) if C16 is not None else 0, p(bias), scale, relu, p(mask),
                                      rup8(N), splits, p(part), _lib.stream_ptr())
    _lib.check(rc, "tb_gemm_bf16x3_ex")
    torch.cuda.synchronize()
    return C, C16, ref


# (M, N, K, layout, splits, epi, BLOCK_N): M / N / K tails, N = 519 (the LSTM's H + 7 over a 128 multiple)
CASES = [
    (300, 24, 200, "kk", 1, 1, 32),
    (129, 50, 520, "kk", 1, 2, 64),
    (1000, 519, 200, "kk", 1, 0, 64),
    (2592, 519, 520, "kk", 1, 1, 128),
    (300, 519, 136, "km", 1, 1, 64),
    (2592, 519, 520, "km", 1, 2, 128),
    (2592, 519, 136, "mm", 1, 2, 128),
    (260, 130, 300, "mm", 1, 1, 64),
    (300, 200, 700, "mm", 2, 1, 64),
    (520, 519, 1000, "mm", 3, 0, 128),
    (2076, 519, 2592, "mm", 4, 1, 64),
]


@pytest.mark.parametrize("M,N,K,layout,splits,epi,bn", CASES)
def test_split_gemm_every_tile_vs_fp64(M, N, K, layout, splits, epi, bn):
    assert block_n(M, N, splits, layout != "kk") == bn
    C, C16, ref = gemm(M, N, K, layout, splits, epi)
    tol = S.tolerance(K, ref.scale, ref.value, extra=ref.extra)
    assert torch.isfinite(C).all()
    err, miss = S.excess(C, ref.value, tol), S.excess(ref.dropped_lo, ref.value, tol)
    assert err <= 1.0, "max |err| / tol = %.3g" % err
    assert miss >= 10.0, "the reference without a lo product is only %.3g x the tolerance" % miss
    if C16 is not None:  # hi + lo planes of the bf16 output carry the fp32 value to 2^-16 of itself
        tol16 = S.tolerance(K, ref.scale, ref.value, rtol=2.0 ** -16 + 2.0 ** -20, extra=ref.extra)
        err16 = S.excess(S.value(C16[0, :, :N], C16[1, :, :N]), ref.value, tol16)
        assert err16 <= 1.0, "bf16 planes: max |err| / tol = %.3g" % err16


@pytest.mark.parametrize("N,K,layout,epi", [(519, 520, "kk", 1), (519, 2076, "km", 2), (512, 3136, "kk", 0)])
def test_tile_width_changes_no_bit(N, K, layout, epi):
    """Rows [0, 300) of a 2592-row product (128-column tiles) equal those of a 300-row call (64-column tiles)."""
    assert block_n(2592, N, 1, layout != "kk") == 128 and block_n(300, N, 1, layout != "kk") == 64
    big, big16, _ = gemm(2592, N, K, layout, 1, epi, seed=5)
    small, small16, _ = gemm(300, N, K, layout, 1, epi, seed=5, gen_m=2592)
    assert torch.equal(big[:300], small)
    if big16 is not None:
        assert torch.equal(big16[:, :300], small16)


def test_split_lstm_bench_shape_vs_fp64():
    """tb_lstm_forward / tb_lstm_backward, bf16x3, at B = 32, H = 519, 81 steps: y, dx and every parameter gradient."""
    from torchbeast_b200 import _lib
    from torchbeast_b200 import lstm as tl
    T1, B, In, H, L = 81, 32, 519, 519, 2
    torch.manual_seed(0)
    ref = torch.nn.LSTM(In, H, num_layers=L).double().cuda()
    m = tl.LSTM(In, H, L, precision="bf16x3")
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    rs = np.random.RandomState(1)
    nd = (rs.rand(T1, B) > 0.05).astype(np.float64)
    x64 = torch.from_numpy(rs.randn(T1, B, In) * 0.5).cuda().requires_grad_(True)
    h064, c064 = (torch.from_numpy(rs.randn(L, B, H) * 0.1).cuda() for _ in range(2))
    dy64 = torch.from_numpy(rs.randn(T1, B, H) / T1 ** 0.5).cuda()
    nd64 = torch.from_numpy(nd).cuda()
    state, ys = (h064, c064), []
    for t in range(T1):
        state = tuple(nd64[t].view(1, -1, 1) * s for s in state)
        yt, state = ref(x64[t:t + 1], state)
        ys.append(yt)
    y64 = torch.cat(ys)
    y64.backward(dy64)

    lib, p = _lib.lib(), _lib.ptr
    prec = tl.PRECISIONS["bf16x3"]
    x, ndf, h0, c0, dy = (t.detach().float().contiguous() for t in (x64, nd64, h064, c064, dy64))
    arr = lambda ts: ctypes.cast(m._ptr_array(ts), ctypes.c_void_p)
    params = [q.detach().contiguous() for q in m._plist()]
    ws = torch.empty(lib.tb_lstm_workspace_bytes(T1, B, In, H, L, prec), dtype=torch.uint8, device="cuda")
    y, hN, cN = torch.empty(T1, B, H, device="cuda"), torch.empty(L, B, H, device="cuda"), torch.empty(L, B, H, device="cuda")
    _lib.check(lib.tb_lstm_forward(p(x), p(ndf), p(h0), p(c0), arr(params), T1, B, In, H, L, prec, p(ws), p(y), p(hN),
                                   p(cN), _lib.stream_ptr()), "tb_lstm_forward")
    dx, grads = torch.empty_like(x), [torch.empty_like(q) for q in params]
    _lib.check(lib.tb_lstm_backward(p(dy), p(x), p(ndf), arr(params), arr(grads), T1, B, In, H, L, prec, p(ws), p(dx),
                                    _lib.stream_ptr()), "tb_lstm_backward")
    torch.cuda.synchronize()

    def rel(a, b):
        a, b = a.double(), b.detach().double()
        return float((a - b).norm() / b.norm().clamp_min(1e-30))

    assert rel(y, y64) < 3e-4, rel(y, y64)
    assert rel(dx, x64.grad) < 3e-4, rel(dx, x64.grad)
    for (n, q), gq in zip(ref.named_parameters(), grads):
        assert rel(gq, q.grad) < 3e-4, (n, rel(gq, q.grad))
