"""The path at other action-space sizes than the fixtures' A=6 (Atari games have 3..18 actions): the LSTM width is
H = 512 + 1 + A, so this moves every recurrence tile size, the heads' output count (A+1 = 19 needs three accumulator
passes) and the fused loss's A-templated kernel.  Network forward and backward for fixed cotangents against the fp64
oracle (oracle/learner_torch.py, autograd): fp32 backend to 1e-4 relative L2, bf16 backend to the mixed-precision
tolerance of test_learner_bf16_gpu.py.  B=5 / T=6 also exercise partial row tiles."""
import numpy as np
import pytest
import torch

from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


# (A, use_lstm, B): B = 5 exercises partial row tiles; B = 40 and 70 leave the cooperative recurrence kernels (they need
# B <= 32): 40 runs the fp32 persistent forward + per-step backward, 70 the per-step kernels both ways (ADVICE r1: the
# large-batch fallbacks were not exercised by any test); A = 18 makes H = 531 > 528, outside the split wavefront kernels
@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16x3"])
@pytest.mark.parametrize("A,use_lstm,B", [(3, True, 5), (18, True, 5), (18, False, 5), (6, True, 40), (6, True, 70)])
def test_forward_backward_other_action_spaces(A, use_lstm, B, precision):
    from torchbeast_b200 import monobeast
    T, seed = (6, 11 + A) if B == 5 else (3, 50 + B)
    batch = LT.synthetic_batch(T, B, A, seed=seed)
    params = LT.random_params(LT.atarinet_param_shapes(A, use_lstm), seed=seed + 100)
    model = monobeast.AtariNet((4, 84, 84), A, use_lstm, precision=precision)
    res = model.load_state_dict(params, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    state = ()
    if use_lstm:
        rs = np.random.RandomState(seed + 7)
        state = tuple(torch.from_numpy(rs.randn(2, B, 512 + A + 1).astype(np.float32) * 0.1) for _ in range(2))
    p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
    ol, ob, ostate = LT.atarinet_forward(p64, batch["frame"], batch["reward"], batch["done"], batch["last_action"],
                                         tuple(s.double() for s in state), A)
    rs = np.random.RandomState(0)
    w1 = torch.from_numpy(rs.randn(*ol.shape)); w2 = torch.from_numpy(rs.randn(*ob.shape))
    names = list(p64)
    ref = dict(zip(names, torch.autograd.grad((ol * w1).sum() + (ob * w2).sum(), [p64[n] for n in names])))
    cb = {k: v.cuda() for k, v in batch.items()}
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    ftol = 1e-2 if precision == "bf16" else 1e-4
    assert rel(out.policy_logits.cpu().double(), ol.detach()) < ftol
    assert rel(out.baseline.cpu().double(), ob.detach()) < ftol
    for a, b in zip(out.core_state, ostate):
        assert rel(a.cpu().double(), b.detach()) < ftol
    model.learner_backward(w1.float().cuda().contiguous(), w2.float().cuda().contiguous())
    report = {}
    for n, p in model.named_parameters():
        got = p.grad.cpu().double()
        cos = float((got * ref[n]).sum() / (got.norm() * ref[n].norm()).clamp_min(1e-30))
        report[n] = (round(rel(got, ref[n]), 5), round(cos, 6))
    if precision == "fp32":
        bad = {n: v for n, v in report.items() if v[0] >= 1e-3}   # ReLU ties can flip single units (test_learner_gpu.py)
    elif precision == "bf16x3":
        bad = {n: v for n, v in report.items() if v[0] >= 6e-3}   # split-bf16: fp32-grade products, more threshold flips
    else:
        # bf16: same mechanism as test_learner_bf16_gpu.py (ReLU sign flips of pre-activations within 2^-9 of zero switch
        # whole gradient paths, error ~ sqrt(flip fraction)); with only N = 35 frames a handful of flips weighs more than in
        # the fixtures, hence 0.2 / 0.98 here instead of 0.12 / 0.995 (conv1 at A=18 without LSTM is the tightest case)
        bad = {n: v for n, v in report.items() if v[0] >= 0.2 or v[1] <= 0.98}
    assert not bad, (bad, report)
