"""GPU: gradients through the recurrent state (tb_lstm_backward_state) and the autograd forward of the standalone LSTM.

The reference is float64 torch.nn.LSTM stepped with the done-reset (monobeast.py:603-611):
    for t: state = state * notdone_t;  y_t, state = lstm(x_t, state)
with loss <y, dy> + <hN, dhN> + <cN, dcN>, so dL/dh0 and dL/dc0 carry the notdone_0 mask.  Every recurrence kind
tb_lstm_plan can choose is covered (the shapes pinned by test_lstm_abi_gpu.test_lstm_plan); tolerances are relative L2 as
in test_lstm_abi_gpu."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_lstm_abi_gpu import BF16_GRAD_TOL

pytestmark = pytest.mark.gpu

TOL = {"fp32": 1e-4, "bf16x3": 3e-4, "bf16": BF16_GRAD_TOL}


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def make_lstm(In, H, layers, precision, seed=0):
    from torchbeast_b200 import lstm as tl
    torch.manual_seed(seed)
    ref = torch.nn.LSTM(In, H, num_layers=layers).double().cuda()
    m = tl.LSTM(In, H, layers, precision=precision)
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
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
        nd[T1 - 1, min(1, B - 1)] = 0.0   # column 0 when it is the only one
    return dict(x=d(rs.randn(T1, B, In) * 0.5), notdone=d(nd), h0=d(rs.randn(layers, B, H) * 0.1),
                c0=d(rs.randn(layers, B, H) * 0.1), dy=d(rs.randn(T1, B, H) / T1 ** 0.5), dhN=d(rs.randn(layers, B, H)),
                dcN=d(rs.randn(layers, B, H)))


def reference(ref, pb):
    """y, hN, cN and the gradients of x, h0, c0 (parameter gradients accumulate into ref's .grad)."""
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


# (T1, B, In, H, layers, precision, backward kind): every kind lstm_plan chooses, at the shapes test_lstm_plan pins
KIND_CASES = [
    (9, 5, 519, 519, 2, "fp32", "persistent"),
    (601, 128, 512, 512, 1, "fp32", "step"),            # BASELINE configs[4]
    (9, 40, 257, 256, 1, "fp32", "step"),
    (1, 40, 257, 256, 1, "fp32", "step"),               # T1 = 1: the first step is also step 0
    (9, 5, 519, 519, 2, "bf16", "wave_bf16"),
    (9, 5, 600, 519, 2, "bf16", "persistent_mma"),
    (9, 8, 257, 256, 1, "bf16", "persistent_mma"),
    (9, 32, 519, 519, 2, "bf16x3", "wave_split"),       # AtariNet's core at bench.py's batch
    (9, 5, 519, 519, 2, "bf16x3", "wave_split"),
    (1, 16, 519, 519, 2, "bf16x3", "wave_split"),
    (9, 8, 257, 256, 1, "bf16x3", "cluster"),           # ResNet's core, one m16 row tile
    (9, 27, 257, 256, 1, "bf16x3", "cluster"),          # two m16 row tiles
    (9, 3, 257, 256, 2, "bf16x3", "persistent"),
]


@pytest.mark.parametrize("T1,B,In,H,layers,precision,kind", KIND_CASES)
def test_state_grads_vs_torch(T1, B, In, H, layers, precision, kind):
    ref, m = make_lstm(In, H, layers, precision)
    assert m.plan(B)[1] == kind
    pb = problem(T1, B, In, H, layers)
    y_ref, (hN_ref, cN_ref), dx_ref, dh0_ref, dc0_ref = reference(ref, pb)
    f = lambda k: pb[k].float().requires_grad_(k in ("x", "h0", "c0"))
    x, h0, c0, nd = f("x"), f("h0"), f("c0"), f("notdone")
    y, (hN, cN) = m(x, (h0, c0), nd)
    torch.autograd.backward([y, hN, cN], [pb["dy"].float(), pb["dhN"].float(), pb["dcN"].float()])
    tol = TOL[precision]
    for name, a, b in (("dx", x.grad, dx_ref), ("dh0", h0.grad, dh0_ref), ("dc0", c0.grad, dc0_ref)):
        assert rel(a, b) < tol, (name, rel(a, b))
    for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert rel(p.grad, q.grad) < tol, (n, rel(p.grad, q.grad))
    # a column that starts an episode at t = 0 never saw h0 / c0
    assert torch.all(h0.grad[:, 0] == 0) and torch.all(c0.grad[:, 0] == 0)
    assert torch.all(h0.grad[:, 1:].abs().sum(-1) > 0)


def _abi_call(m, pb, ports, fill=None):
    """tb_lstm_forward, then tb_lstm_backward (ports None) or tb_lstm_backward_state with the given ports; returns the
    outputs ([dx] + parameter gradients + [y, hN, cN]) and the number of kernel launches of the backward call.  With
    `fill` (a byte value) the workspace starts out filled with it instead of holding whatever torch.empty left."""
    from torchbeast_b200 import _lib
    from torchbeast_b200.lstm import PRECISIONS
    lib, p = _lib.lib(), _lib.ptr
    x, nd, h0, c0, dy = (pb[k].float().contiguous() for k in ("x", "notdone", "h0", "c0", "dy"))
    T1, B, In = x.shape
    H, L, prec = m.hidden_size, m.num_layers, PRECISIONS[m.precision]
    arr = lambda ts: ctypes.cast(m._ptr_array(ts), ctypes.c_void_p)
    params = [q.detach().contiguous() for q in m._plist()]
    ws = torch.empty(lib.tb_lstm_workspace_bytes(T1, B, In, H, L, prec), dtype=torch.uint8, device="cuda")
    if fill is not None:
        ws.fill_(fill)
    y, hN, cN = torch.empty(T1, B, H, device="cuda"), torch.empty(L, B, H, device="cuda"), torch.empty(L, B, H, device="cuda")
    _lib.check(lib.tb_lstm_forward(p(x), p(nd), p(h0), p(c0), arr(params), T1, B, In, H, L, prec, p(ws), p(y), p(hN), p(cN),
                                   _lib.stream_ptr()), "tb_lstm_forward")
    dx, grads = torch.empty_like(x), [torch.empty_like(q) for q in params]
    torch.cuda.synchronize()
    n0 = lib.tb_launch_count()
    if ports is None:
        rc = lib.tb_lstm_backward(p(dy), p(x), p(nd), arr(params), arr(grads), T1, B, In, H, L, prec, p(ws), p(dx),
                                  _lib.stream_ptr())
    else:
        rc = lib.tb_lstm_backward_state(p(dy), p(x), p(nd), arr(params), arr(grads), T1, B, In, H, L, prec, p(ws), p(dx),
                                        *[p(t) for t in ports], _lib.stream_ptr())
    _lib.check(rc, "tb_lstm_backward")
    n = lib.tb_launch_count() - n0
    torch.cuda.synchronize()
    return [dx] + grads + [y, hN, cN], n


@pytest.mark.parametrize("T1,B,In,H,layers,precision,kind", [c for c in KIND_CASES if c[0] == 9])
def test_null_ports_change_nothing(T1, B, In, H, layers, precision, kind):
    _, m = make_lstm(In, H, layers, precision)
    assert m.plan(B)[1] == kind
    pb = problem(T1, B, In, H, layers)
    base, n_base = _abi_call(m, pb, None)
    null, n_null = _abi_call(m, pb, (None, None, None, None))
    assert n_null == n_base
    for a, b in zip(null, base):
        assert torch.equal(a, b)


@pytest.mark.parametrize("T,B,In,H,layers,precision", [
    (7, 4, 33, 48, 2, "fp32"),
    (7, 32, 519, 519, 2, "bf16x3"),
    (7, 8, 257, 256, 1, "bf16x3"),
])
def test_autograd_forward_vs_torch_lstm(T, B, In, H, layers, precision):
    """notdone=None is torch.nn.LSTM: outputs and gradients to x, h0, c0 and the parameters; also with the loss on h_n
    only (no gradient on the output) and with hx=None."""
    ref, m = make_lstm(In, H, layers, precision)
    pb = problem(T, B, In, H, layers)
    tol = TOL[precision]
    for case in ("full", "h_n only", "hx=None"):
        ref.zero_grad()
        m.zero_grad()
        leaves = lambda src: [src[k].clone().requires_grad_(True) for k in ("x", "h0", "c0")]
        rx, rh0, rc0 = leaves(pb)
        ox, oh0, oc0 = leaves({k: pb[k].float() for k in ("x", "h0", "c0")})
        if case == "hx=None":
            ry, (rhN, rcN) = ref(rx)
            oy, (ohN, ocN) = m(ox)
        else:
            ry, (rhN, rcN) = ref(rx, (rh0, rc0))
            oy, (ohN, ocN) = m(ox, (oh0, oc0))
        for a, b in ((oy, ry), (ohN, rhN), (ocN, rcN)):
            assert rel(a, b) < tol, (case, rel(a, b))
        if case == "h_n only":
            torch.autograd.backward(rhN, pb["dhN"])
            torch.autograd.backward(ohN, pb["dhN"].float())
        else:
            torch.autograd.backward([ry, rhN, rcN], [pb["dy"], pb["dhN"], pb["dcN"]])
            torch.autograd.backward([oy, ohN, ocN], [pb["dy"].float(), pb["dhN"].float(), pb["dcN"].float()])
        pairs = [("dx", ox.grad, rx.grad)]
        if case != "hx=None":
            pairs += [("dh0", oh0.grad, rh0.grad), ("dc0", oc0.grad, rc0.grad)]
        else:
            assert oh0.grad is None and oc0.grad is None
        pairs += [(n, p.grad, q.grad) for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters())]
        for name, a, b in pairs:
            assert rel(a, b) < tol, (case, name, rel(a, b))


def test_two_forwards_backward_in_reverse_order():
    ref, m = make_lstm(519, 519, 2, "bf16x3")
    p1, p2 = problem(9, 32, 519, 519, 2, seed=1), problem(5, 32, 519, 519, 2, seed=2)
    refs = [reference(ref, pb) for pb in (p1, p2)]   # parameter gradients of both accumulate into ref
    outs = []
    for pb in (p1, p2):
        x, h0, c0 = (pb[k].float().requires_grad_(True) for k in ("x", "h0", "c0"))
        outs.append(((x, h0, c0), m(x, (h0, c0), pb["notdone"].float())))
    for pb, (_, (y, (hN, cN))) in reversed(list(zip((p1, p2), outs))):
        torch.autograd.backward([y, hN, cN], [pb[k].float() for k in ("dy", "dhN", "dcN")])
    for ((x, h0, c0), _), (_, _, dx, dh0, dc0) in zip(outs, refs):
        for name, a, b in (("dx", x.grad, dx), ("dh0", h0.grad, dh0), ("dc0", c0.grad, dc0)):
            assert rel(a, b) < TOL["bf16x3"], (name, rel(a, b))
    for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert rel(p.grad, q.grad) < TOL["bf16x3"], (n, rel(p.grad, q.grad))


@pytest.mark.parametrize("T,B,In,H,layers,precision", [
    (40, 32, 519, 519, 2, "bf16x3"),    # AtariNet's core: the wavefront kernels
    (40, 8, 257, 256, 1, "bf16x3"),     # ResNet's core: the cluster kernels
    (40, 5, 519, 519, 2, "fp32"),       # persistent fp32
    (24, 40, 257, 256, 1, "fp32"),      # step kernels
])
def test_truncated_bptt_matches_one_call(T, B, In, H, layers, precision):
    """Two chained calls on the halves of a sequence, no detach between them, backpropagated together, against one call
    over the whole sequence."""
    _, m = make_lstm(In, H, layers, precision)
    pb = problem(T, B, In, H, layers)
    nd = pb["notdone"].float()
    dys = [pb[k].float() for k in ("dy", "dhN", "dcN")]
    grads = []
    for chained in (False, True):
        m.zero_grad()
        x, h0, c0 = (pb[k].float().requires_grad_(True) for k in ("x", "h0", "c0"))
        if chained:
            k = T // 2
            y1, s1 = m(x[:k], (h0, c0), nd[:k])
            y2, (hN, cN) = m(x[k:], s1, nd[k:])
            y = torch.cat([y1, y2])
        else:
            y, (hN, cN) = m(x, (h0, c0), nd)
        torch.autograd.backward([y, hN, cN], dys)
        grads.append([y, hN, cN, x.grad, h0.grad, c0.grad] + [p.grad.clone() for p in m.parameters()])
    names = ["y", "hN", "cN", "dx", "dh0", "dc0"] + [n for n, _ in m.named_parameters()]
    for name, a, b in zip(names, grads[1], grads[0]):
        assert rel(a, b) < TOL[precision], (name, rel(a, b))
