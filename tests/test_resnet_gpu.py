"""GPU parity of the IMPALA ResNet path (torchbeast_b200.polybeast_learner: Net + learn) against the
golden fixtures produced by the reference's own polybeast_learner.learn (tests/golden/learn_resnet_*.npz)
and the torch-CPU oracle; mirrors /root/reference/tests/polybeast_learn_function_test.py and
polybeast_net_test.py.  fp32 backend: tight tolerances; bf16 tensor-core backend: the mixed-precision
tolerances explained in test_learner_bf16_gpu.py."""
import types
import unittest.mock as mock

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests.common import golden

pytestmark = pytest.mark.gpu

CASES = ["learn_resnet_T4_B2.npz", "learn_resnet_lstm_T4_B2.npz"]


def build(fname, precision="fp32"):
    from torchbeast_b200 import optim, polybeast_learner
    g = golden(fname)
    T, B, A, seed, use_lstm = [int(x) for x in g["meta"]]
    batch = LT.synthetic_batch(T, B, A, seed=seed, with_last_action=False)
    params = LT.random_params(LT.resnet_param_shapes(A, bool(use_lstm)), seed=seed + 100)
    model = polybeast_learner.Net(A, bool(use_lstm), precision=precision)
    actor = polybeast_learner.Net(A, bool(use_lstm), precision=precision)
    res = model.load_state_dict(params, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    state = ()
    if use_lstm:
        rs = np.random.RandomState(seed + 7)
        state = tuple(torch.from_numpy(rs.randn(1, B, 256).astype(np.float32) * 0.1) for _ in range(2))
    opt = optim.RMSprop(model, lr=0.00048, momentum=0, eps=0.01, alpha=0.99)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 1.0)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006,
                                  grad_norm_clipping=float(g["clip"]), unroll_length=T, batch_size=B, learner_device="cuda")
    return g, model, actor, batch, params, state, opt, sched, flags


def queue_of(batch, state):
    env = (batch["frame"], batch["reward"], batch["done"], batch["episode_step"], batch["episode_return"])
    agent = (batch["action"], batch["policy_logits"], batch["baseline"])
    q = mock.MagicMock()
    q.__iter__.return_value = iter([((env, agent), state)])
    q.size.return_value = 0
    return q


@pytest.mark.parametrize("fname", CASES)
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_net_forward_matches_reference(fname, precision):
    g, model, actor, batch, params, state, opt, sched, flags = build(fname, precision)
    model.eval()
    cb = {k: v.cuda() for k, v in batch.items()}
    with torch.no_grad():
        (action, logits, baseline), new_state = model(dict(frame=cb["frame"], reward=cb["reward"], done=cb["done"]),
                                                      tuple(s.cuda() for s in state))
    np.testing.assert_allclose(logits.cpu().numpy(), g["policy_logits"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(baseline.cpu().numpy(), g["baseline"], rtol=1e-4, atol=1e-4)
    T1, B = batch["frame"].shape[:2]
    assert tuple(action.shape) == (T1, B) and tuple(logits.shape) == (T1, B, 6) and tuple(baseline.shape) == (T1, B)
    ol, ob, ostate = LT.resnet_forward(params, batch["frame"], batch["reward"], batch["done"], state)
    for a, b in zip(new_state, ostate):
        np.testing.assert_allclose(a.cpu().numpy(), b.numpy(), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("fname", CASES)
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_learn_matches_reference(fname, precision):
    from torchbeast_b200 import polybeast_learner
    g, model, actor, batch, params, state, opt, sched, flags = build(fname, precision)
    stats, plogger = {}, mock.Mock()
    polybeast_learner.learn(flags, queue_of(batch, state), model, actor, opt, sched, stats, plogger)
    plogger.log.assert_called_once()
    assert stats["step"] == flags.unroll_length * flags.batch_size
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(stats[k], float(g[k]), rtol=5e-5, atol=5e-5, err_msg=k)
        assert stats[k] != 0.0
    total = 0.0
    for n, p in model.named_parameters():
        gr = p.grad.detach().cpu()
        total += float((gr.double() ** 2).sum())
        scale = max(float(g["grad_stats/" + n][2]), 1e-6)
        # split-bf16: conv outputs carry ~5e-6 relative rounding, enough to flip a handful of max-pool argmax / ReLU
        # decisions in this tiny case; every flip moves the gradients upstream of it by ~1e-3 of their norm while tensors
        # with no flip upstream agree to 1e-5 (tools/resnet_flips.py) - same bounds as the T=80 baseline tests
        gatol, nrtol = (5e-4, 2e-3) if precision == "fp32" else (1.5e-2, 2e-2)
        np.testing.assert_allclose(gr.flatten()[:16].numpy(), g["grad_head/" + n], rtol=5e-3, atol=gatol * scale, err_msg=n)
        np.testing.assert_allclose(float(gr.double().norm()), float(g["grad_stats/" + n][2]), rtol=nrtol, atol=1e-6, err_msg=n)
        # RMSprop divides by sqrt(v) + eps: an element whose gradient moved by a max-pool / ReLU tie flipping under the
        # split-bf16 rounding (~1e-6 relative pre-activations) moves by up to lr / sqrt(1 - alpha) = 4.8e-3; same bound as
        # tests/test_learner_baseline_gpu.py
        patol = 1e-5 if precision == "fp32" else 5e-4
        np.testing.assert_allclose(p.detach().cpu().flatten()[:16].numpy(), g["param_head/" + n], rtol=1e-4, atol=patol, err_msg=n)
        assert float(gr.abs().sum()) > 0, n  # every gradient non-zero (reference test :157-179)
    np.testing.assert_allclose(np.sqrt(total), float(g["clipped_grad_norm"]), rtol=1e-3)
    for (n, a), (_, b) in zip(actor.named_parameters(), model.named_parameters()):
        assert torch.equal(a, b), n  # actor weights == learner weights (reference test :108-119)


@pytest.mark.parametrize("fname", CASES)
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_backward_vs_oracle_fixed_cotangents(fname, precision):
    g, model, actor, batch, params, state, opt, sched, flags = build(fname, precision)
    p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
    ol, ob, _ = LT.resnet_forward(p64, batch["frame"], batch["reward"], batch["done"], tuple(s.double() for s in state))
    rs = np.random.RandomState(0)
    w1 = torch.from_numpy(rs.randn(*ol.shape)); w2 = torch.from_numpy(rs.randn(*ob.shape))
    names = list(p64)
    ref = dict(zip(names, torch.autograd.grad((ol * w1).sum() + (ob * w2).sum(), [p64[n] for n in names])))
    cb = {k: v.cuda() for k, v in batch.items()}
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    rel = lambda a, b: float((a - b).norm() / b.norm().clamp_min(1e-30))
    ftol = {"fp32": 1e-5, "bf16x3": 3e-5, "bf16": 2e-2}[precision]
    assert rel(out.policy_logits.cpu().double(), ol.detach()) < ftol
    assert rel(out.baseline.cpu().double(), ob.detach()) < ftol
    model.learner_backward(w1.float().cuda().contiguous(), w2.float().cuda().contiguous())
    report = {}
    for n, p in model.named_parameters():
        got = p.grad.cpu().double()
        cos = float((got * ref[n]).sum() / (got.norm() * ref[n].norm()).clamp_min(1e-30))
        report[n] = (round(rel(got, ref[n]), 5), round(cos, 6))
    # split-bf16 ("bf16x3"): hi.hi + hi.lo + lo.hi products, ~2^-17 relative each: 1e-5 where no max-pool / ReLU decision
    # flips upstream; in this 10-frame case ONE flipped ReLU / argmax moves a gradient tensor by up to ~1e-2 of its norm and
    # which elements flip depends on the summation order (tools/resnet_flips.py).  So: every tensor within 3e-2 with
    # cosine > 0.9995, and the MEDIAN tensor within 5e-3 (plain bf16 operands sit at 2e-2 .. 2e-1 on every tensor)
    lim = {"fp32": (1e-4, 0.999999), "bf16x3": (3e-2, 0.9995), "bf16": (0.2, 0.98)}[precision]
    bad = {n: v for n, v in report.items() if v[0] >= lim[0] or v[1] <= lim[1]}
    if precision == "bf16x3":
        med = float(np.median([v[0] for v in report.values()]))
        assert med < 5e-3, (med, report)
    assert not bad, (bad, report)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_learn_step_at_one_gpu_shard_of_config4(precision):
    """BASELINE configs[3] (ResNet + LSTM, T=80, B=64 over 8 GPUs) -> one GPU's shard: T=80, B=8, against the fixture the
    reference's polybeast_learner.learn produced at that size (learn_resnet_lstm_T80_B8.npz): outputs, V-trace targets,
    losses, 4096 strided gradient samples per tensor, updated parameters.  Same tolerance structure as
    tests/test_learner_baseline_gpu.py; both parity-grade backends (fp32 SIMT and split-bf16 tensor-core GEMMs)."""
    from tests.common import sample_index
    from torchbeast_b200 import learner, polybeast_learner
    g, model, actor, batch, params, state, opt, sched, flags = build("learn_resnet_lstm_T80_B8.npz", precision)
    cb = {k: v.cuda() for k, v in batch.items()}
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    np.testing.assert_allclose(out.policy_logits.cpu().numpy(), g["policy_logits"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out.baseline.cpu().numpy(), g["baseline"], rtol=1e-5, atol=1e-5)
    loss = learner.impala_loss_fwd_bwd(cb["policy_logits"][1:], out.policy_logits[:-1], cb["action"][1:], cb["reward"][1:],
                                       cb["done"][1:], out.baseline[:-1], out.baseline[-1])
    np.testing.assert_allclose(loss.vs.cpu().numpy(), g["vs"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(loss.pg_advantages.cpu().numpy(), g["pg_advantages"], rtol=1e-5, atol=1e-5)
    stats = {}
    polybeast_learner.learn(flags, queue_of(batch, state), model, actor, opt, sched, stats, mock.Mock())
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(stats[k], float(g[k]), rtol=1e-5, atol=1e-5, err_msg=k)
    assert stats["step"] == 80 * 8
    for n, p in model.named_parameters():
        gr = p.grad.detach().cpu().flatten()
        idx = torch.from_numpy(sample_index(gr.numel()))
        ref = torch.from_numpy(g["grad_sample/" + n]).double()
        got = gr[idx].double()
        rel = float((got - ref).norm() / ref.norm().clamp_min(1e-30))
        worst = float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        assert rel < 6e-3 and worst < 1.5e-2, (n, rel, worst)
        np.testing.assert_allclose(p.detach().cpu().flatten()[idx].numpy(), g["param_sample/" + n], rtol=1e-4, atol=5e-4, err_msg=n)
    for (n, a), (_, b) in zip(actor.named_parameters(), model.named_parameters()):
        assert torch.equal(a, b), n


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_results_do_not_depend_on_stale_workspace_contents(precision):
    """The workspace comes from torch.empty: whatever a previous owner left there (here: all bytes 0xFF = NaN patterns in
    fp32 and bf16) must not reach the results - every byte a kernel reads is written earlier in the same pass.  Caught a
    real hazard: the weight-gradient kernel read 15 pixels of slack behind the last image plane, multiplied by exact
    zeros (0 * NaN)."""
    g, model, actor, batch, params, state, opt, sched, flags = build("learn_resnet_lstm_T4_B2.npz", precision)
    cb = {k: v.cuda() for k, v in batch.items()}
    st = tuple(s.cuda() for s in state)
    rs = np.random.RandomState(1)
    runs = []
    for fill in (None, 255, 0):
        if fill is not None:
            model._ws.fill_(fill)
        out = model.learner_forward(cb, st)
        w1 = torch.from_numpy(rs.randn(*out.policy_logits.shape)).float().cuda() if not runs else runs[0][2]
        w2 = torch.from_numpy(rs.randn(*out.baseline.shape)).float().cuda() if not runs else runs[0][3]
        model.learner_backward(w1.contiguous(), w2.contiguous())
        runs.append((out.policy_logits.clone(), model.flat_grad.clone(), w1, w2))
    for logits, grads, _, _ in runs[1:]:
        assert torch.isfinite(grads).all()
        assert torch.equal(logits, runs[0][0]) and torch.equal(grads, runs[0][1])
