"""GPU: the split-bf16 two-layer backward wavefront (lstm2_bwd_wave_split_kernel) at the sequence ends.

The kernel hands its gate gradients and its partial products through 2-slot buffers in L2, and its lower-layer role runs
one wave step behind the upper one.  Unrolls of 1 to 4 steps make those buffers wrap and put that lag across the first
and the last step, with gradients arriving at the final state (dhN / dcN).  The reference is float64 torch.nn.LSTM with the
done-reset, as in test_lstm_state_grad_gpu; the backward must also be bit-identical from run to run (fixed summation order,
no atomics)."""
import numpy as np
import pytest
import torch

from tests.test_lstm_state_grad_gpu import TOL, _abi_call, make_lstm, problem, reference, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [5, 32])
def test_plan_is_wave_split(B):
    _, m = make_lstm(519, 519, 2, "bf16x3")
    assert m.plan(B) == ("wave_split", "wave_split")


@pytest.mark.parametrize("T1,B", [(1, 32), (2, 32), (3, 32), (4, 32), (3, 17)])
def test_short_unrolls_vs_torch(T1, B):
    ref, m = make_lstm(519, 519, 2, "bf16x3")
    assert m.plan(B)[1] == "wave_split"
    pb = problem(T1, B, 519, 519, 2)
    _, _, dx_ref, dh0_ref, dc0_ref = reference(ref, pb)
    f = lambda k: pb[k].float().requires_grad_(k in ("x", "h0", "c0"))
    x, h0, c0, nd = f("x"), f("h0"), f("c0"), f("notdone")
    y, (hN, cN) = m(x, (h0, c0), nd)
    torch.autograd.backward([y, hN, cN], [pb["dy"].float(), pb["dhN"].float(), pb["dcN"].float()])
    tol = TOL["bf16x3"]
    for name, a, b in (("dx", x.grad, dx_ref), ("dh0", h0.grad, dh0_ref), ("dc0", c0.grad, dc0_ref)):
        assert rel(a, b) < tol, (name, rel(a, b))
    for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert rel(p.grad, q.grad) < tol, (n, rel(p.grad, q.grad))


@pytest.mark.parametrize("T1", [3, 9])
def test_backward_bit_identical_across_runs(T1):
    _, m = make_lstm(519, 519, 2, "bf16x3")
    pb = problem(T1, 32, 519, 519, 2)
    ports = lambda: (pb["dhN"].float().contiguous(), pb["dcN"].float().contiguous(),
                     torch.full((2, 32, 519), np.nan, device="cuda"), torch.full((2, 32, 519), np.nan, device="cuda"))
    first, second = ports(), ports()
    a, _ = _abi_call(m, pb, first)
    b, _ = _abi_call(m, pb, second)
    for u, v in zip(a + list(first[2:]), b + list(second[2:])):
        assert torch.equal(u, v)
