"""GPU: stacks of more than two layers, run as a chain of two-layer segments (tb_lstm_* with layers > 2).

The reference is float64 torch.nn.LSTM of the same depth stepped with the done-reset (monobeast.py:603-611):
    for t: state = state * notdone_t;  y_t, state = lstm(x_t, state)
with loss <y, dy> + <hN, dhN> + <cN, dcN>.  Tolerances are the ones test_lstm_state_grad_gpu uses for each precision."""
import numpy as np
import pytest
import torch

from tests.test_lstm_state_grad_gpu import TOL

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def make_lstm(In, H, layers, precision, seed=0):
    from torchbeast_b200 import lstm as tl
    torch.manual_seed(seed)
    ref = torch.nn.LSTM(In, H, num_layers=layers).double().cuda()
    m = tl.LSTM(In, H, layers, precision=precision)
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()}, strict=True)
    return ref, m


def problem(T1, B, In, H, layers, seed=1):
    """float64 CUDA inputs; column 0 starts an episode at t = 0, column 1 resets at the last step (T1 > 1), every other
    column sees h0 / c0."""
    rs = np.random.RandomState(seed)
    d = lambda a: torch.from_numpy(a).cuda()
    nd = (rs.rand(T1, B) > 0.1).astype(np.float64)
    nd[0, 0] = 0.0
    nd[0, 1:] = 1.0
    if T1 > 1:
        nd[T1 - 1, 1] = 0.0
    return dict(x=d(rs.randn(T1, B, In) * 0.5), notdone=d(nd), h0=d(rs.randn(layers, B, H) * 0.1),
                c0=d(rs.randn(layers, B, H) * 0.1), dy=d(rs.randn(T1, B, H) / T1 ** 0.5), dhN=d(rs.randn(layers, B, H)),
                dcN=d(rs.randn(layers, B, H)))


def reference(ref, pb):
    """y, (hN, cN) and the gradients of x, h0, c0 (parameter gradients accumulate into ref's .grad)."""
    x, h0, c0 = (pb[k].clone().requires_grad_(True) for k in ("x", "h0", "c0"))
    state, ys = (h0, c0), []
    for t in range(x.shape[0]):
        nd = pb["notdone"][t].view(1, -1, 1)
        state = tuple(nd * s for s in state)
        y, state = ref(x[t:t + 1], state)
        ys.append(y)
    y = torch.cat(ys)
    torch.autograd.backward([y, state[0], state[1]], [pb["dy"], pb["dhN"], pb["dcN"]])
    return y, state, x.grad, h0.grad, c0.grad


def leaves(pb):
    return [pb[k].float().requires_grad_(True) for k in ("x", "h0", "c0")]


def run(m, pb, x, h0, c0):
    y, (hN, cN) = m(x, (h0, c0), pb["notdone"].float())
    torch.autograd.backward([y, hN, cN], [pb[k].float() for k in ("dy", "dhN", "dcN")])
    return y, hN, cN


P, PS, S, C = ("persistent",) * 2, ("persistent", "step"), ("step",) * 2, ("cluster",) * 2
WB, WS, MMA = ("wave_bf16",) * 2, ("wave_split",) * 2, ("persistent_mma",) * 2

# (T1, B, In, H, layers, precision, plan_layers(B))
DEEP_CASES = [
    (9, 5, 519, 519, 3, "fp32", [P] * 3),
    (9, 5, 519, 519, 4, "fp32", [P] * 4),
    (9, 5, 519, 519, 5, "fp32", [P] * 5),
    (9, 40, 257, 256, 3, "fp32", [PS] * 3),
    (9, 70, 96, 128, 4, "fp32", [S] * 4),
    # first segment: forward wavefront, backward persistent_mma (In > H); the pair above: the wavefront both ways
    (9, 5, 600, 519, 4, "bf16", [("wave_bf16", "persistent_mma")] * 2 + [WB] * 2),
    (9, 5, 600, 519, 5, "bf16", [("wave_bf16", "persistent_mma")] * 2 + [WB] * 2 + [MMA]),
    (9, 32, 519, 519, 4, "bf16x3", [WS] * 4),
    (9, 5, 519, 519, 5, "bf16x3", [WS] * 4 + [P]),
    (9, 32, 600, 519, 4, "bf16x3", [P] * 2 + [WS] * 2),            # In != H: only the upper pair is a wavefront
    (9, 8, 257, 256, 3, "bf16x3", [("cluster", "persistent")] * 2 + [C]),  # a lone cluster top layer
    (1, 16, 519, 519, 3, "bf16x3", [WS] * 2 + [P]),                 # T1 = 1
    (1, 40, 257, 256, 4, "fp32", [PS] * 4),
    (601, 128, 512, 512, 3, "fp32", [S] * 3),                       # BASELINE configs[4], three layers
]


@pytest.mark.parametrize("T1,B,In,H,layers,precision,kinds", DEEP_CASES)
def test_deep_vs_torch(T1, B, In, H, layers, precision, kinds):
    ref, m = make_lstm(In, H, layers, precision)
    assert m.plan_layers(B) == kinds
    pb = problem(T1, B, In, H, layers)
    y_ref, (hN_ref, cN_ref), dx_ref, dh0_ref, dc0_ref = reference(ref, pb)
    x, h0, c0 = leaves(pb)
    y, hN, cN = run(m, pb, x, h0, c0)
    tol = TOL[precision]
    pairs = [("y", y, y_ref), ("hN", hN, hN_ref), ("cN", cN, cN_ref), ("dx", x.grad, dx_ref), ("dh0", h0.grad, dh0_ref),
             ("dc0", c0.grad, dc0_ref)]
    pairs += [(n, p.grad, q.grad) for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters())]
    for name, a, b in pairs:
        assert rel(a, b) < tol, (name, rel(a, b))
    # a column that starts an episode at t = 0 never saw h0 / c0, in any layer
    assert torch.all(h0.grad[:, 0] == 0) and torch.all(c0.grad[:, 0] == 0)
    assert torch.all(h0.grad[:, 1:].abs().sum(-1) > 0)


@pytest.mark.parametrize("T1,B,In,H,precision", [
    (9, 5, 519, 519, "fp32"),
    (9, 40, 257, 256, "fp32"),
    (9, 5, 600, 519, "bf16"),       # side-stream GEMMs below, a wavefront tail above
    (9, 32, 519, 519, "bf16x3"),    # two split wavefront segments
    (9, 8, 257, 256, "bf16x3"),
])
def test_four_layers_equal_two_chained_pairs(T1, B, In, H, precision):
    """A four-layer module is bit for bit two two-layer modules with the same weights, chained through autograd with the
    lower module's h_n / c_n in the loss."""
    from torchbeast_b200 import lstm as tl
    _, deep = make_lstm(In, H, 4, precision)
    sd = deep.state_dict()
    lo, hi = tl.LSTM(In, H, 2, precision=precision), tl.LSTM(H, H, 2, precision=precision)
    lo.load_state_dict({k: sd[k] for k in lo.state_dict()}, strict=True)
    hi.load_state_dict({k: sd[k[:-1] + str(int(k[-1]) + 2)] for k in hi.state_dict()}, strict=True)
    pb = problem(T1, B, In, H, 4)
    nd = pb["notdone"].float()
    dys = [pb[k].float() for k in ("dy", "dhN", "dcN")]

    x, h0, c0 = leaves(pb)
    y, hN, cN = run(deep, pb, x, h0, c0)
    cx, ch0, cc0 = leaves(pb)
    y1, (h1, c1) = lo(cx, (ch0[:2], cc0[:2]), nd)
    cy, (h2, c2) = hi(y1, (ch0[2:], cc0[2:]), nd)
    chN, ccN = torch.cat([h1, h2]), torch.cat([c1, c2])
    torch.autograd.backward([cy, chN, ccN], dys)

    pairs = [("y", y, cy), ("hN", hN, chN), ("cN", cN, ccN), ("dx", x.grad, cx.grad), ("dh0", h0.grad, ch0.grad),
             ("dc0", c0.grad, cc0.grad)]
    chained = dict(lo.named_parameters())
    chained.update({n[:-1] + str(int(n[-1]) + 2): p for n, p in hi.named_parameters()})
    pairs += [(n, p.grad, chained[n].grad) for n, p in deep.named_parameters()]
    for name, a, b in pairs:
        assert torch.equal(a, b), name


@pytest.mark.parametrize("B,In,H,layers,precision", [
    (5, 519, 519, 1, "fp32"), (5, 519, 519, 2, "fp32"), (40, 257, 256, 1, "fp32"), (5, 519, 519, 2, "bf16"),
    (5, 600, 519, 2, "bf16"), (8, 257, 256, 1, "bf16"), (32, 519, 519, 2, "bf16x3"), (8, 257, 256, 1, "bf16x3"),
    (3, 257, 256, 2, "bf16x3"), (40, 257, 256, 1, "bf16x3"),
])
def test_plan_layers_agrees_with_plan(B, In, H, layers, precision):
    from torchbeast_b200 import lstm as tl
    m = tl.LSTM(In, H, layers, precision=precision)
    assert m.plan_layers(B) == [m.plan(B)] * layers


def test_torch_state_dict_loads_strictly():
    from torchbeast_b200 import lstm as tl
    ref = torch.nn.LSTM(100, 64, num_layers=4).cuda()
    m = tl.LSTM(100, 64, 4)
    m.load_state_dict(ref.state_dict(), strict=True)
    for (n, p), (rn, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert n == rn and torch.equal(p, q)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_truncated_bptt_three_layers(precision):
    """Two chained calls on the halves of a sequence at three layers, backpropagated together, against one call over the
    whole sequence: the gradient crosses from the second call into the first through every layer's state."""
    T, B, In, H, L = 24, 8, 519, 519, 3
    _, m = make_lstm(In, H, L, precision)
    pb = problem(T, B, In, H, L)
    nd = pb["notdone"].float()
    dys = [pb[k].float() for k in ("dy", "dhN", "dcN")]
    out = []
    for chained in (False, True):
        m.zero_grad()
        x, h0, c0 = leaves(pb)
        if chained:
            k = T // 2
            y1, s1 = m(x[:k], (h0, c0), nd[:k])
            y2, (hN, cN) = m(x[k:], s1, nd[k:])
            y = torch.cat([y1, y2])
        else:
            y, (hN, cN) = m(x, (h0, c0), nd)
        torch.autograd.backward([y, hN, cN], dys)
        out.append([y, hN, cN, x.grad, h0.grad, c0.grad] + [p.grad.clone() for p in m.parameters()])
    names = ["y", "hN", "cN", "dx", "dh0", "dc0"] + [n for n, _ in m.named_parameters()]
    for name, a, b in zip(names, out[1], out[0]):
        assert rel(a, b) < TOL[precision], (name, rel(a, b))
