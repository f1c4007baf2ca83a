"""GPU: every recurrence kind at the edges of its geometry, against float64 torch.nn.LSTM.

The other LSTM tests run the tensor-core recurrences at H = 256 and 519 only, and both avoid the edges the launch code
creates: an idle CTA in the last 2-CTA cluster of the split forward wavefront, a partial last k-group in the split
backward, padding columns of H mod 16 other than 0 and 7, batches of 1 and at the template switches, inputs narrower than
8 and narrower than H.  Each case here asserts the kinds tb_lstm_plan chooses on an H100 (132 SMs) and compares y, hN, cN,
dx, dh0, dc0 and every parameter gradient with the tolerances of test_lstm_state_grad_gpu (the float64 harness is shared
with it), with non-zero dhN / dcN and resets at t = 0 and t = T1-1.  Further down: the workspace is scratch only (a
NaN-filled one gives bit-identical results) and hidden sizes past the backward's limit are rejected before any launch."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_lstm_state_grad_gpu import TOL, _abi_call, make_lstm, problem, reference, rel

pytestmark = pytest.mark.gpu

# ---- geometry of the split wavefront kernels (torchbeast_b200/csrc/lstm.cu), restated -----------------------------------
K_SPLIT = 3   # kSplitK: k16 steps per warp (forward k-slice) and per backward k-group


def split_fwd_ctas(H):
    """wave_fwd_split_launch: kStepUnits = 4 hidden units per CTA, rounded up to whole 2-CTA clusters."""
    return ((H + 3) // 4 + 1) & ~1


def split_idle_fwd_cta(H):
    """lstm2_fwd_wave_split: nctas = ceil(H / 4) CTAs own units; the padding CTA of the last cluster owns none."""
    return split_fwd_ctas(H) - (H + 3) // 4 == 1


def split_bwd_groups(H):
    """wave_bwd_split_groups: ceil(ceil(H / 16) / kSplitK) k-groups of the backward's recurrent product."""
    return ((H + 15) // 16 + K_SPLIT - 1) // K_SPLIT


def split_partial_group(H):
    """The last k-group holds fewer than kSplitK k16 steps."""
    return (H + 15) // 16 % K_SPLIT != 0


EDGES = {
    "single group": lambda H: split_bwd_groups(H) == 1 and split_partial_group(H) and not split_idle_fwd_cta(H),
    "one full group": lambda H: split_bwd_groups(H) == 1 and not split_partial_group(H) and not split_idle_fwd_cta(H),
    "idle cta, partial group": lambda H: split_idle_fwd_cta(H) and split_partial_group(H),
    "partial group": lambda H: split_partial_group(H) and not split_idle_fwd_cta(H),
    "idle cta, full groups": lambda H: split_idle_fwd_cta(H) and not split_partial_group(H),
    "largest": lambda H: True,
}

# The largest H tb_lstm_plan keeps on each tensor-core kind on an H100 (132 SMs), at every B <= 32 with In = H: all three
# run ceil(H / 4) CTAs that must be co-resident at one per SM, so 4 * 132 = 528.  For wave_split that is also the
# ceil(H / 16) <= 33 k16-step bound (11 warps x kSplitK); mma_fits' own bound (624) is not reached.
WAVE_SPLIT_MAX_H = WAVE_BF16_MAX_H = MMA_MAX_H = 528


def test_split_geometry_restated():
    """The restated formulas agree with the shapes the other wave_split tests pin: H = 519 is 130 forward CTAs (no idle
    one) and 11 full k-groups."""
    assert split_fwd_ctas(519) == 130 and not split_idle_fwd_cta(519)
    assert split_bwd_groups(519) == 11 and not split_partial_group(519)
    assert split_fwd_ctas(100) == 26 and split_idle_fwd_cta(100)
    assert split_bwd_groups(100) == 3 and split_partial_group(100)


def _check(T1, B, In, H, layers, precision, kinds):
    ref, m = make_lstm(In, H, layers, precision)
    assert m.plan(B) == kinds
    pb = problem(T1, B, In, H, layers)
    y_ref, (hN_ref, cN_ref), dx_ref, dh0_ref, dc0_ref = reference(ref, pb)
    f = lambda k: pb[k].float().requires_grad_(k in ("x", "h0", "c0"))
    x, h0, c0, nd = f("x"), f("h0"), f("c0"), f("notdone")
    y, (hN, cN) = m(x, (h0, c0), nd)
    torch.autograd.backward([y, hN, cN], [pb["dy"].float(), pb["dhN"].float(), pb["dcN"].float()])
    tol = TOL[precision]
    pairs = [("y", y, y_ref), ("hN", hN, hN_ref), ("cN", cN, cN_ref), ("dx", x.grad, dx_ref), ("dh0", h0.grad, dh0_ref),
             ("dc0", c0.grad, dc0_ref)]
    pairs += [(n, p.grad, q.grad) for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters())]
    for name, a, b in pairs:
        assert torch.isfinite(a).all(), name
        assert rel(a, b) < tol, (name, rel(a, b))
    # column 0 starts an episode at t = 0: it never saw h0 / c0
    assert torch.all(h0.grad[:, 0] == 0) and torch.all(c0.grad[:, 0] == 0)


# ---- wave_split: bf16x3, two layers, In = H --------------------------------------------------------------------------
@pytest.mark.parametrize("H,B,edge", [
    (8, 1, "single group"),
    (16, 17, "single group"),
    (48, 32, "one full group"),
    (100, 5, "idle cta, partial group"),
    (500, 9, "idle cta, partial group"),
    (256, 32, "partial group"),
    (513, 32, "idle cta, full groups"),     # H = 1 (mod 16): one real unit in the last k16 step
    (WAVE_SPLIT_MAX_H, 32, "largest"),      # 132 forward CTAs, 11 full groups
])
def test_wave_split_edges(H, B, edge):
    assert EDGES[edge](H)
    _check(7, B, H, H, 2, "bf16x3", ("wave_split", "wave_split"))


# ---- wave_bf16: bf16, two layers ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,B,In,kinds", [
    (8, 1, 8, ("wave_bf16", "wave_bf16")),
    (100, 17, 100, ("wave_bf16", "wave_bf16")),
    (512, 5, 512, ("wave_bf16", "wave_bf16")),
    (256, 32, 37, ("wave_bf16", "wave_bf16")),          # In < H: the backward wavefront too
    (100, 8, 300, ("wave_bf16", "persistent_mma")),     # In > H: the backward runs per layer
    (WAVE_BF16_MAX_H, 32, WAVE_BF16_MAX_H, ("wave_bf16", "wave_bf16")),
])
def test_wave_bf16_edges(H, B, In, kinds):
    _check(7, B, In, H, 2, "bf16", kinds)


# ---- persistent_mma: bf16, one layer ----------------------------------------------------------------------------------
@pytest.mark.parametrize("H,B", [(8, 1), (100, 16), (MMA_MAX_H, 32)])
def test_persistent_mma_edges(H, B):
    _check(7, B, H, H, 1, "bf16", ("persistent_mma", "persistent_mma"))


# ---- cluster: bf16x3, H = 256 only ------------------------------------------------------------------------------------
@pytest.mark.parametrize("In", [1, 256])
@pytest.mark.parametrize("B", [1, 16, 17, 32])   # one m16 row tile up to B = 16, two above
def test_cluster_batches(B, In):
    _check(7, B, In, 256, 1, "bf16x3", ("cluster", "cluster"))


def test_cluster_forward_two_layers():
    """In != H keeps two layers off wave_split: the cluster forward per layer, the persistent fp32 backward."""
    _check(7, 17, 257, 256, 2, "bf16x3", ("cluster", "persistent"))


# ---- fp32 recurrences, and bf16 above the tensor-core range ------------------------------------------------------------
@pytest.mark.parametrize("H,B,In,precision,kinds", [
    (100, 33, 100, "fp32", ("persistent", "step")),     # persistent forward takes B <= 64, backward B <= 32
    (100, 64, 100, "fp32", ("persistent", "step")),
    (8, 32, 8, "fp32", ("persistent", "persistent")),
    (700, 4, 700, "fp32", ("step", "step")),            # TB_LSTM_MAX_HIDDEN
    (700, 200, 700, "fp32", ("step", "step")),
    (1, 3, 1, "fp32", ("persistent", "persistent")),
    (100, 65, 100, "fp32", ("step", "step")),
    (640, 8, 640, "bf16", ("step", "step")),            # past mma_fits: fp32 recurrence under bf16 projections
])
def test_fp32_recurrence_edges(H, B, In, precision, kinds):
    _check(7, B, In, H, 1, precision, kinds)


# ---- narrow inputs (the bf16 operand is padded to ld16(In) = 8) -------------------------------------------------------
@pytest.mark.parametrize("In", [1, 3, 9])
@pytest.mark.parametrize("H,layers,precision,kinds", [
    (100, 1, "fp32", ("persistent", "persistent")),
    (100, 2, "bf16", ("wave_bf16", "wave_bf16")),
    (256, 1, "bf16x3", ("cluster", "cluster")),
])
def test_narrow_inputs(In, H, layers, precision, kinds):
    _check(7, 8, In, H, layers, precision, kinds)


# ---- one- and two-step unrolls on every tensor-core kind ----------------------------------------------------------------
@pytest.mark.parametrize("T1", [1, 2])
@pytest.mark.parametrize("B,In,H,layers,precision,kinds", [
    (5, 100, 100, 2, "bf16x3", ("wave_split", "wave_split")),
    (17, 100, 100, 2, "bf16", ("wave_bf16", "wave_bf16")),
    (16, 100, 100, 1, "bf16", ("persistent_mma", "persistent_mma")),
    (17, 1, 256, 1, "bf16x3", ("cluster", "cluster")),
])
def test_short_unrolls(T1, B, In, H, layers, precision, kinds):
    _check(T1, B, In, H, layers, precision, kinds)


# ---- the workspace is scratch: stale contents change nothing ----------------------------------------------------------
@pytest.mark.parametrize("B,In,H,layers,precision,kind", [
    (5, 100, 100, 2, "bf16x3", "wave_split"),
    (17, 100, 100, 2, "bf16", "wave_bf16"),
    (16, 100, 100, 1, "bf16", "persistent_mma"),
    (17, 257, 256, 1, "bf16x3", "cluster"),
    (8, 100, 100, 1, "fp32", "persistent"),
    (65, 100, 100, 1, "fp32", "step"),
])
def test_stale_workspace_bit_identical(B, In, H, layers, precision, kind):
    """0xFF bytes read as NaN in fp32 and in bf16: a kernel that multiplies any stale padding, even by zero, poisons its
    outputs.  Two runs on a NaN-filled workspace and one on a zeroed one must agree bit for bit."""
    _, m = make_lstm(In, H, layers, precision)
    assert m.plan(B) == (kind, kind)
    pb = problem(7, B, In, H, layers)
    runs = []
    for fill in (0xFF, 0xFF, 0x00):
        ports = (pb["dhN"].float().contiguous(), pb["dcN"].float().contiguous(),
                 torch.full((layers, B, H), np.nan, device="cuda"), torch.full((layers, B, H), np.nan, device="cuda"))
        out, _ = _abi_call(m, pb, ports, fill=fill)
        runs.append(out + list(ports[2:]))
    for r in runs:
        assert all(torch.isfinite(t).all() for t in r)
    for other in runs[1:]:
        for u, v in zip(runs[0], other):
            assert torch.equal(u, v)


# ---- hidden sizes the backward cannot run -----------------------------------------------------------------------------
def test_hidden_size_above_the_bound_is_rejected():
    """H = 701 (fp32, B = 4) used to run forward and then fail in the backward; every entry now rejects it first."""
    from torchbeast_b200 import _lib
    from torchbeast_b200 import lstm as tl
    lib, p = _lib.lib(), _lib.ptr
    H, B, T1 = tl.MAX_HIDDEN + 1, 4, 3
    assert lib.tb_lstm_workspace_bytes(T1, B, H, H, 1, 0) == 0
    m = tl.LSTM(H, H)
    with pytest.raises(_lib.TorchBeastB200Error, match="hidden size 701 above 700"):
        m.plan(B)
    with pytest.raises(_lib.TorchBeastB200Error, match="hidden size 701 above 700"):
        m(torch.zeros(T1, B, H, device="cuda"))
    x, nd = torch.zeros(T1, B, H, device="cuda"), torch.ones(T1, B, device="cuda")
    s = torch.zeros(1, B, H, device="cuda")
    params = [q.detach() for q in m._plist()]
    arr = ctypes.cast(m._ptr_array(params), ctypes.c_void_p)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    n0 = lib.tb_launch_count()
    assert lib.tb_lstm_forward(p(x), p(nd), p(s), p(s), arr, T1, B, H, H, 1, 0, p(ws), p(x), p(s), p(s), _lib.stream_ptr()) != 0
    assert lib.tb_lstm_backward(p(x), p(x), p(nd), arr, arr, T1, B, H, H, 1, 0, p(ws), p(x), _lib.stream_ptr()) != 0
    assert "hidden size 701 above 700" in lib.tb_last_error().decode()
    assert lib.tb_launch_count() == n0
