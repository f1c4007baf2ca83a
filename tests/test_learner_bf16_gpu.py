"""GPU: the bf16 tensor-core backend (precision="bf16": wgmma GEMMs with bf16 operands and fp32
accumulation for the conv/fc trunk and the LSTM projections) against the fp64 oracle.
bf16 carries 8 mantissa bits (unit roundoff 2^-9 ~ 2e-3), so this is a mixed-precision tolerance,
stated per quantity: learner outputs relative L2 error < 1e-2, losses rtol 3e-2, and -
for fixed cotangents - every parameter gradient relative L2 error < 0.12 with cosine similarity > 0.995.
tools/bf16_report.py prints the per-tensor errors.  The conv/fc error is NOT GEMM rounding (that is ~3e-3): a bf16 forward flips the sign of the ~0.2% of
ReLU pre-activations that sit within 2^-9 of zero, and each flip switches a whole gradient path, so the
L2 error is ~sqrt(flip fraction).  Any reduced-precision forward (incl. the reference's own TF32 cuDNN
path on GPU) has this property; the same script shows the fp32 backend at 5e-7.  The fp32 backend holds
the tight parity contract in test_learner_gpu.py."""
import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests.test_learner_gpu import build_case, flags_for, to_cuda

pytestmark = pytest.mark.gpu

CASES = ["learn_atari_T4_B2.npz", "learn_atari_T20_B4.npz", "learn_atari_lstm_T4_B2.npz", "learn_atari_lstm_T20_B4.npz"]


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


@pytest.mark.parametrize("fname", CASES)
def test_bf16_forward_and_backward_vs_oracle(fname):
    """Network forward and backward in isolation: the SAME fixed cotangents (w1, w2) are pushed through
    the fp64 oracle (autograd) and through the bf16 CUDA backward, so the comparison measures the kernels'
    mixed-precision error and not the loss's own sensitivity to the forward values (vs - V cancels)."""
    g, model, actor, batch, params, state, opt, sched = build_case(fname, precision="bf16")
    A = int(g["meta"][2])
    p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
    ol, ob, _ = LT.atarinet_forward(p64, batch["frame"], batch["reward"], batch["done"], batch["last_action"],
                                    tuple(s.double() for s in state), A)
    rs = np.random.RandomState(0)
    w1 = torch.from_numpy(rs.randn(*ol.shape)); w2 = torch.from_numpy(rs.randn(*ob.shape))
    names = list(p64)
    ref_grads = dict(zip(names, torch.autograd.grad((ol * w1).sum() + (ob * w2).sum(), [p64[n] for n in names])))
    cb = to_cuda(batch)
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    assert rel(out.policy_logits.cpu().double(), ol.detach()) < 1e-2
    assert rel(out.baseline.cpu().double(), ob.detach()) < 1e-2
    model.learner_backward(w1.float().cuda().contiguous(), w2.float().cuda().contiguous())
    report = {}
    for n, p in model.named_parameters():
        ref = ref_grads[n]
        got = p.grad.cpu().double()
        cos = float((got * ref).sum() / (got.norm() * ref.norm()).clamp_min(1e-30))
        report[n] = (round(rel(got, ref), 4), round(cos, 5))
    bad = {n: v for n, v in report.items() if v[0] >= 0.12 or v[1] <= 0.995}
    assert not bad, (bad, report)


@pytest.mark.parametrize("fname", CASES)
def test_bf16_losses_vs_oracle(fname):
    from torchbeast_b200 import learner
    g, model, actor, batch, params, state, opt, sched = build_case(fname, precision="bf16")
    p64 = {k: v.double() for k, v in params.items()}
    o = LT.learner_step(p64, batch, tuple(s.double() for s in state), net="atari", update=False)
    cb = to_cuda(batch)
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    loss = learner.impala_loss_fwd_bwd(cb["policy_logits"][1:], out.policy_logits[:-1], cb["action"][1:], cb["reward"][1:],
                                       cb["done"][1:], out.baseline[:-1], out.baseline[-1])
    np.testing.assert_allclose(float(loss.losses[1]), float(o["baseline_loss"]), rtol=3e-2)
    np.testing.assert_allclose(float(loss.losses[2]), float(o["entropy_loss"]), rtol=3e-2)
    np.testing.assert_allclose(float(loss.losses[3]), float(o["total_loss"]), rtol=3e-2, atol=3e-2 * float(o["baseline_loss"]))
    assert rel(loss.vs.cpu().double(), o["vs"]) < 2e-2


@pytest.mark.parametrize("fname", ["learn_atari_T20_B4.npz", "learn_atari_lstm_T20_B4.npz"])
def test_bf16_learn_step_runs_and_is_deterministic(fname):
    from torchbeast_b200 import monobeast
    outs = []
    for _ in range(2):
        g, model, actor, batch, params, state, opt, sched = build_case(fname, precision="bf16")
        flags = flags_for(g)
        cb = to_cuda(batch)
        st = tuple(s.cuda() for s in state)
        s1 = monobeast.learn(flags, actor, model, cb, st, opt, sched)
        s2 = monobeast.learn(flags, actor, model, cb, st, opt, sched)
        np.testing.assert_allclose(s1["total_loss"], float(g["total_loss"]), rtol=3e-2, atol=0.5)
        outs.append((s1["total_loss"], s2["total_loss"], model.flat_params.clone()))
        assert torch.equal(actor.flat_params, model.flat_params)
    assert outs[0][0] == outs[1][0] and outs[0][1] == outs[1][1] and torch.equal(outs[0][2], outs[1][2])
