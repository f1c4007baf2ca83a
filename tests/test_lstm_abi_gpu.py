"""GPU: the standalone LSTM C ABI (tb_lstm_forward / tb_lstm_backward, SURVEY 8(b) B3) with hidden size, layers and batch
as parameters, against torch.nn.LSTM stepped with the reference's done-reset (monobeast.py:603-611):
    for t: state = state * notdone_t;  y_t, state = lstm(x_t, state)
Cases: AtariNet's core (2 x 519), ResNet's core (257 -> 256), and BASELINE configs[4] "long-unroll stress T=600 B=128,
LSTM hidden=512" at fp32 (forward 1e-4; backward gradients relative L2 1e-4 through 600 dependent steps).
test_lstm_plan pins which recurrence implementation each case runs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def torch_reference(ref, x, notdone, h0, c0, dy):
    x = x.clone().requires_grad_(True)
    state = (h0, c0)
    ys = []
    for t in range(x.shape[0]):
        nd = notdone[t].view(1, -1, 1)
        state = tuple(nd * s for s in state)
        y, state = ref(x[t:t + 1], state)
        ys.append(y)
    y = torch.cat(ys)
    y.backward(dy)
    return y.detach(), state, x.grad


@pytest.mark.parametrize("B,In,H,layers,precision,fwd,bwd", [
    (5, 519, 519, 2, "fp32", "persistent", "persistent"),
    (128, 512, 512, 1, "fp32", "step", "step"),                     # BASELINE configs[4]
    (40, 257, 256, 1, "fp32", "persistent", "step"),
    (5, 519, 519, 2, "bf16", "wave_bf16", "wave_bf16"),
    (5, 600, 519, 2, "bf16", "wave_bf16", "persistent_mma"),        # the backward wavefront needs In <= H
    (8, 257, 256, 1, "bf16", "persistent_mma", "persistent_mma"),
    (40, 257, 256, 1, "bf16", "persistent", "step"),
    (32, 519, 519, 2, "bf16x3", "wave_split", "wave_split"),         # AtariNet's core at bench.py's batch
    (5, 519, 519, 2, "bf16x3", "wave_split", "wave_split"),
    (8, 257, 256, 1, "bf16x3", "cluster", "cluster"),               # ResNet's core, one m16 row tile
    (27, 257, 256, 1, "bf16x3", "cluster", "cluster"),              # two m16 row tiles (16 < B <= 32)
    (3, 257, 256, 2, "bf16x3", "cluster", "persistent"),            # the cluster backward runs one layer only
    (40, 257, 256, 1, "bf16x3", "persistent", "step"),
])
def test_lstm_plan(B, In, H, layers, precision, fwd, bwd):
    from torchbeast_b200 import lstm as tl
    assert tl.LSTM(In, H, layers, precision=precision).plan(B) == (fwd, bwd)


# bf16 (precision 1) bounds, relative L2: about 3x the largest error over the three bf16 cases below, measured on an
# H100 80GB HBM3 (700 W power limit)
BF16_FWD_TOL = 7e-3    # y / hN / cN; largest measured 2.38e-3
BF16_GRAD_TOL = 1.1e-2  # dx and every parameter gradient; largest measured 3.75e-3


@pytest.mark.parametrize("T1,B,In,H,layers,precision", [
    (9, 5, 519, 519, 2, "fp32"),
    (9, 5, 519, 519, 2, "bf16x3"),
    (9, 5, 519, 519, 2, "bf16"),
    (9, 5, 600, 519, 2, "bf16"),         # the upper layer's weight gradients on the side stream beside the lower recurrence
    (7, 40, 257, 256, 1, "fp32"),
    (7, 40, 257, 256, 1, "bf16x3"),
    (7, 8, 257, 256, 1, "bf16"),
    (81, 8, 257, 256, 1, "bf16x3"),      # the IMPALA ResNet's LSTM at one GPU's shard of configs[3]
    (33, 27, 257, 256, 1, "bf16x3"),
    (12, 3, 257, 256, 2, "bf16x3"),      # two layers of H = 256
    (601, 128, 512, 512, 1, "fp32"),     # BASELINE configs[4]
])
def test_lstm_abi_vs_torch(T1, B, In, H, layers, precision):
    from torchbeast_b200 import lstm as tl
    torch.manual_seed(0)
    ref = torch.nn.LSTM(In, H, num_layers=layers).double()
    m = tl.LSTM(In, H, layers, precision=precision)
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    rs = np.random.RandomState(1)
    x = torch.from_numpy(rs.randn(T1, B, In)) * 0.5
    notdone = torch.from_numpy((rs.rand(T1, B) > 0.02).astype(np.float64))
    h0 = torch.from_numpy(rs.randn(layers, B, H)) * 0.1
    c0 = torch.from_numpy(rs.randn(layers, B, H)) * 0.1
    dy = torch.from_numpy(rs.randn(T1, B, H)) / T1 ** 0.5
    y_ref, (hN_ref, cN_ref), dx_ref = torch_reference(ref, x, notdone, h0, c0, dy)
    y, (hN, cN) = m.forward_unroll(x.float().cuda(), notdone.float().cuda(), (h0.float().cuda(), c0.float().cuda()))

    def rel(a, b):
        return float((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-30))
    if precision == "bf16":
        for name, a, b in (("y", y, y_ref), ("hN", hN, hN_ref.detach()), ("cN", cN, cN_ref.detach())):
            assert rel(a, b) < BF16_FWD_TOL, (name, rel(a, b))
    else:
        np.testing.assert_allclose(y.cpu().numpy(), y_ref.numpy(), rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(hN.cpu().numpy(), hN_ref.detach().numpy(), rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(cN.cpu().numpy(), cN_ref.detach().numpy(), rtol=1e-4, atol=1e-4)
    dx = m.backward_unroll(dy.float().cuda())
    tol = {"fp32": 1e-4, "bf16x3": 3e-4, "bf16": BF16_GRAD_TOL}[precision]
    assert rel(dx, dx_ref) < tol, rel(dx, dx_ref)
    for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert rel(p.grad, q.grad) < tol, (n, rel(p.grad, q.grad))
