"""GPU parity AT THE BASELINE CONFIG (BASELINE.json configs[1]: AtariNet +-LSTM, T=80, B=32 - the size bench.py
runs) against fixtures produced by the reference's own monobeast.learn (tests/golden/learn_atari*_T80_B32.npz,
oracle/make_golden.py --baseline-config): learner outputs, V-trace targets (vs, pg_advantages), the four losses,
clipped gradients (4096 strided samples per tensor + norms) and the updated parameters, for the DEFAULT backend
("bf16x3": split-bf16 tensor-core products - what bench.py times) and the fp32 SIMT anchor.

Tolerances - the SAME for both backends:
  * learner outputs, vs, pg_advantages: 1e-5 absolute + 1e-5 relative (10x inside north_star's 1e-4); the four
    losses rtol 1e-5.
  * gradients (4096 strided samples per tensor): relative L2 error < 6e-3 and max |err| < 1.5e-2 x max |ref| per
    tensor, norms within 2e-3.  This is NOT product rounding (the LSTM / head gradients, which see no ReLU, agree to
    1e-5): at 2592 frames x 21 k ReLU units some pre-activations sit within fp32 rounding of zero, any two fp32-grade
    implementations disagree on those signs, and every flip switches a gradient path - for the exact-fp32 SIMT backend as
    much as for bf16x3 (tools/parity_report.py prints the per-tensor errors of both backends).
  * updated parameters: atol 5e-4.  The first RMSprop step divides by sqrt(0.01 g^2) + 0.01, i.e. moves every weight by
    ~0.048 x g for small g, so a 5e-3 absolute gradient difference becomes 2.5e-4 in the weight."""
import numpy as np
import pytest
import torch

from tests.common import sample_index
from tests.test_learner_gpu import build_case, flags_for, to_cuda

pytestmark = pytest.mark.gpu

CASES = ["learn_atari_lstm_T80_B32.npz", "learn_atari_T80_B32.npz"]
PRECISIONS = ["bf16x3", "fp32"]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("fname", CASES)
def test_outputs_and_vtrace_targets(fname, precision):
    from torchbeast_b200 import learner
    g, model, actor, batch, params, state, opt, sched = build_case(fname, precision=precision)
    cb = to_cuda(batch)
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    np.testing.assert_allclose(out.policy_logits.cpu().numpy(), g["policy_logits"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out.baseline.cpu().numpy(), g["baseline"], rtol=1e-5, atol=1e-5)
    loss = learner.impala_loss_fwd_bwd(cb["policy_logits"][1:], out.policy_logits[:-1], cb["action"][1:], cb["reward"][1:],
                                       cb["done"][1:], out.baseline[:-1], out.baseline[-1])
    np.testing.assert_allclose(loss.vs.cpu().numpy(), g["vs"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(loss.pg_advantages.cpu().numpy(), g["pg_advantages"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(float(loss.losses[3]), float(g["total_loss"]), rtol=1e-5)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("fname", CASES)
def test_learn_step_matches_reference(fname, precision):
    from torchbeast_b200 import monobeast
    g, model, actor, batch, params, state, opt, sched = build_case(fname, precision=precision)
    assert model.precision == precision
    flags = flags_for(g)
    stats = monobeast.learn(flags, actor, model, to_cuda(batch), tuple(s.cuda() for s in state), opt, sched)
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(stats[k], float(g[k]), rtol=1e-5, atol=1e-5, err_msg=k)
    total = 0.0
    for n, p in model.named_parameters():
        gr = p.grad.detach().cpu().flatten()
        total += float((gr.double() ** 2).sum())
        idx = torch.from_numpy(sample_index(gr.numel()))
        ref = torch.from_numpy(g["grad_sample/" + n]).double()
        got = gr[idx].double()
        rel = float((got - ref).norm() / ref.norm().clamp_min(1e-30))
        worst = float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        assert rel < 6e-3 and worst < 1.5e-2, (n, rel, worst)
        np.testing.assert_allclose(float(gr.double().norm()), float(g["grad_stats/" + n][2]), rtol=2e-3, atol=1e-6, err_msg=n)
        np.testing.assert_allclose(p.detach().cpu().flatten()[idx].numpy(), g["param_sample/" + n], rtol=1e-4, atol=5e-4,
                                   err_msg=n)
        np.testing.assert_allclose(float(p.detach().double().norm()), float(g["param_stats/" + n][2]), rtol=1e-3, err_msg=n)
    np.testing.assert_allclose(np.sqrt(total), float(g["clipped_grad_norm"]), rtol=1e-4)
    for (n, a), (_, b) in zip(actor.named_parameters(), model.named_parameters()):
        assert torch.equal(a, b), n


def test_default_backend_is_the_parity_backend():
    """bench.py / monobeast.learn run the backend these tests hold to the 1e-4 contract."""
    from torchbeast_b200 import monobeast
    m = monobeast.AtariNet((4, 84, 84), 6, True)
    assert m.precision == "bf16x3"
