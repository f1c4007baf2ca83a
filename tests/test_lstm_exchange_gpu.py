"""GPU: the split (bf16x3) two-layer wavefront, whose forward exchanges h through a slice-blocked buffer fetched with one
1-D bulk copy per warp and group, forward and backward against float64 torch.nn.LSTM.

Every case runs the wave_split plan at H = 519 (bench.py's shape: 130 forward CTAs, 11 full warp slices) or H = 500 (125
forward CTAs; units 500..511 of the last slice are never written by any CTA and must read as zero), at batches on both
sides of the 16-row halves, and unrolls from one step (the acting forward) to bench.py's 81.  Each case also checks that
the results are bit-identical from run to run and with a NaN-filled workspace: the exchange buffer's padding rows and
columns are multiplied by zero weights, so anything but zeros there would change them."""
import numpy as np
import pytest
import torch

from tests.test_lstm_state_grad_gpu import TOL, _abi_call, make_lstm, problem, reference, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("T1", [1, 2, 3, 4, 81])
@pytest.mark.parametrize("H", [500, 519])
@pytest.mark.parametrize("B", [1, 5, 16, 17, 32])
def test_wave_split_exchange_vs_torch(B, H, T1):
    ref, m = make_lstm(H, H, 2, "bf16x3")
    assert m.plan(B) == ("wave_split", "wave_split")
    pb = problem(T1, B, H, H, 2)
    y_ref, (hN_ref, cN_ref), dx_ref, dh0_ref, dc0_ref = reference(ref, pb)
    f = lambda k: pb[k].float().requires_grad_(k in ("x", "h0", "c0"))
    x, h0, c0, nd = f("x"), f("h0"), f("c0"), f("notdone")
    y, (hN, cN) = m(x, (h0, c0), nd)
    torch.autograd.backward([y, hN, cN], [pb["dy"].float(), pb["dhN"].float(), pb["dcN"].float()])
    tol = TOL["bf16x3"]
    pairs = [("y", y, y_ref), ("hN", hN, hN_ref), ("cN", cN, cN_ref), ("dx", x.grad, dx_ref), ("dh0", h0.grad, dh0_ref),
             ("dc0", c0.grad, dc0_ref)]
    pairs += [(n, p.grad, q.grad) for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters())]
    for name, a, b in pairs:
        assert torch.isfinite(a).all(), name
        assert rel(a, b) < tol, (name, rel(a, b))

    # run to run, and a NaN-filled (0xFF) workspace against a zeroed one: bit for bit
    runs = []
    for fill in (0xFF, 0xFF, 0x00):
        ports = (pb["dhN"].float().contiguous(), pb["dcN"].float().contiguous(),
                 torch.full((2, B, H), np.nan, device="cuda"), torch.full((2, B, H), np.nan, device="cuda"))
        out, _ = _abi_call(m, pb, ports, fill=fill)
        runs.append(out + list(ports[2:]))
    for r in runs:
        assert all(torch.isfinite(t).all() for t in r)
    for other in runs[1:]:
        for u, v in zip(runs[0], other):
            assert torch.equal(u, v)
