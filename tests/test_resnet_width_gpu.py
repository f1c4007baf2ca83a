"""IMPALA ResNet with other section widths (channels=(c0, c1, c2), each 16, 32 or 64) on every backend: forward and
backward against the float64 autograd of oracle/learner_torch.resnet_forward (which reads its sizes from the
parameters) at the narrowest and widest rows of the observation range, the default widths bit for bit, the learner,
PopArt, the acting paths, a stale workspace, and the inputs a wide net rejects."""
import gc
import functools
import types
import unittest.mock as mock

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu

A = 6
X2 = (32, 64, 64)
# (16, 64, 32): a 64 -> 32 feat conv, whose input gradient is a 32 -> 64 conv
WIDTHS = [X2, (64, 64, 64), (16, 64, 32)]
SHAPES = [(4, 84, 84), (3, 64, 64), (2, 17, 33), (16, 126, 126)]
FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


@pytest.fixture(autouse=True)
def _collect_graphs():
    yield
    gc.collect()
    torch.cuda.synchronize()


def param_shapes(obs, channels, num_actions=A, use_lstm=False, num_values=1):
    from torchbeast_b200.nets import resnet_param_spec
    return dict(resnet_param_spec(num_actions, use_lstm, num_values, observation_shape=obs, channels=channels))


def obs_batch(obs, T, B, seed):
    batch = LT.synthetic_batch(T, B, A, seed=seed, with_last_action=False)
    rs = np.random.RandomState(seed + 1000)
    batch["frame"] = torch.from_numpy(rs.randint(0, 256, size=(T + 1, B) + tuple(obs)).astype(np.uint8))
    return batch


def make(obs, channels, use_lstm, precision, params=None, **kw):
    from torchbeast_b200 import polybeast_learner
    m = polybeast_learner.Net(A, use_lstm, precision=precision, observation_shape=obs, channels=channels, **kw)
    if params is not None:
        res = m.load_state_dict(params, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
    return m


def lstm_state(B, use_lstm, seed=7):
    if not use_lstm:
        return ()
    rs = np.random.RandomState(seed)
    return tuple(torch.from_numpy(rs.randn(1, B, 256).astype(np.float32) * 0.1) for _ in range(2))


@functools.lru_cache(maxsize=4)
def oracle_case(obs, channels, use_lstm):
    """(params, batch, state, cotangents, float64 outputs, float64 parameter gradients) of a T=2, B=2 case."""
    T, B = 2, 2
    params = LT.random_params(param_shapes(obs, channels, A, use_lstm), seed=sum(obs) + sum(channels) + use_lstm)
    batch = obs_batch(obs, T, B, seed=sum(obs))
    state = lstm_state(B, use_lstm)
    p64 = {k: v.double().requires_grad_(True) for k, v in params.items()}
    ol, ob, _ = LT.resnet_forward(p64, batch["frame"], batch["reward"], batch["done"], tuple(s.double() for s in state), A)
    rs = np.random.RandomState(0)
    w1, w2 = torch.from_numpy(rs.randn(*ol.shape)), torch.from_numpy(rs.randn(*ob.shape))
    names = list(p64)
    grads = torch.autograd.grad((ol * w1).sum() + (ob * w2).sum(), [p64[n] for n in names])
    return params, batch, state, (w1, w2), (ol.detach(), ob.detach()), dict(zip(names, grads))


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("use_lstm", [False, True])
@pytest.mark.parametrize("obs", SHAPES)
@pytest.mark.parametrize("channels", WIDTHS)
def test_forward_backward_vs_float64_oracle(channels, obs, use_lstm, precision):
    params, batch, state, (w1, w2), (ol, ob), ref = oracle_case(obs, channels, use_lstm)
    model = make(obs, channels, use_lstm, precision, params)
    cb = {k: v.cuda() for k, v in batch.items()}
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    logits, baseline = out.policy_logits.cpu().double(), out.baseline.cpu().double()
    assert tuple(logits.shape) == tuple(ol.shape) and tuple(baseline.shape) == tuple(ob.shape)
    if precision == "bf16":   # bf16 activations through convs 2-4x wider than test_resnet_obs_gpu.py's
        assert rel(logits, ol) < 4e-2 and rel(baseline, ob) < 4e-2
    else:
        np.testing.assert_allclose(logits.numpy(), ol.numpy(), rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(baseline.numpy(), ob.numpy(), rtol=1e-4, atol=1e-4)
    model.learner_backward(w1.float().cuda().contiguous(), w2.float().cuda().contiguous())
    got = {n: p.grad.cpu().double() for n, p in model.named_parameters()}
    assert list(got) == list(ref)
    report = {n: (rel(got[n], ref[n]), float((got[n] * ref[n]).sum() / (got[n].norm() * ref[n].norm()).clamp_min(1e-30)))
              for n in ref}
    flat_got = torch.cat([got[n].flatten() for n in ref])
    flat_ref = torch.cat([ref[n].flatten() for n in ref])
    # the tolerances of test_resnet_obs_gpu.py, except where noted: a 64-channel conv sums 2-4x more products per output
    # and per weight-gradient element, and more of them cancel.  Measured on an H100 over these cases: fp32 per tensor
    # at most 4.6e-3 with cosine > 0.99998 (feat_convs.0.0.weight, whose gradient cancels most); bf16 (single-plane
    # operands and activations, not parity-grade) logits 2.5e-3, baseline 2.7e-2, whole gradient up to 0.22 with
    # cosines above 0.96 ((16, 64, 32) at (2, 17, 33))
    if precision == "fp32":
        bad = {n: v for n, v in report.items() if v[0] >= 1e-2 or v[1] <= 0.9999}
    elif precision == "bf16x3":
        assert rel(flat_got, flat_ref) < 6e-3, report
        bad = {n: v for n, v in report.items() if v[0] >= 3e-2 or v[1] <= 0.9995}
    else:
        assert rel(flat_got, flat_ref) < 0.3, report
        assert float(np.median([v[0] for v in report.values()])) < 0.3, report
        bad = {n: v for n, v in report.items() if v[0] >= 0.5 or v[1] <= 0.9}
    assert not bad, (bad, report)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("use_lstm", [False, True])
@pytest.mark.parametrize("obs", [(4, 84, 84), (3, 64, 64)])
def test_default_widths_are_bit_identical(obs, use_lstm, precision):
    """channels=(16, 32, 32) is the model built without `channels`: outputs and gradients bit for bit."""
    params, batch, state, (w1, w2), _, _ = oracle_case(obs, (16, 32, 32), use_lstm)
    runs = []
    for kw in ({}, {"channels": (16, 32, 32)}):
        from torchbeast_b200 import polybeast_learner
        model = polybeast_learner.Net(A, use_lstm, precision=precision, observation_shape=obs, **kw)
        model.load_state_dict(params)
        out = model.learner_forward({k: v.cuda() for k, v in batch.items()}, tuple(s.cuda() for s in state))
        model.learner_backward(w1.float().cuda().contiguous(), w2.float().cuda().contiguous())
        runs.append((out.policy_logits, out.baseline, model.flat_grad.clone()))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def queue_of(batch, state):
    env = (batch["frame"], batch["reward"], batch["done"], batch["episode_step"], batch["episode_return"])
    agent = (batch["action"], batch["policy_logits"], batch["baseline"])
    q = mock.MagicMock()
    q.__iter__.return_value = iter([((env, agent), state)])
    q.size.return_value = 0
    return q


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("use_lstm", [False, True])
def test_polybeast_learn_step_vs_oracle(use_lstm, precision):
    from torchbeast_b200 import optim, polybeast_learner
    obs, T, B = (3, 64, 64), 4, 3
    params = LT.random_params(param_shapes(obs, X2, A, use_lstm), seed=21)
    batch = obs_batch(obs, T, B, seed=22)
    state = lstm_state(B, use_lstm)
    ref = LT.learner_step(params, batch, state, net="resnet", num_actions=A)
    model, actor = make(obs, X2, use_lstm, precision, params), make(obs, X2, use_lstm, precision)
    opt = optim.RMSprop(model, lr=LT.Hyper.learning_rate, momentum=0, eps=LT.Hyper.epsilon, alpha=LT.Hyper.alpha)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 1.0)
    flags = types.SimpleNamespace(unroll_length=T, batch_size=B, learner_device="cuda", **FLAGS)
    stats = {}
    polybeast_learner.learn(flags, queue_of(batch, state), model, actor, opt, sched, stats, mock.Mock())
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(stats[k], float(ref[k]), rtol=1e-4, atol=1e-4, err_msg=k)
    # (fp32: an element whose gradient moved by 1e-3 relative moves by up to lr / sqrt(1 - alpha) under RMSprop too)
    patol = 5e-4
    for n, p in model.named_parameters():
        np.testing.assert_allclose(p.detach().cpu().numpy(), ref["params"][n].numpy(), rtol=1e-4, atol=patol, err_msg=n)
    assert torch.equal(actor.flat_params, model.flat_params)


def _learn_runs(obs, graph, steps, num_tasks=None, T=6, B=4, beta=0.0):
    from torchbeast_b200 import learner, optim
    model = make(obs, X2, True, None, num_tasks=num_tasks)
    actor = make(obs, X2, True, None, num_tasks=num_tasks)
    model.reset_parameters_like_torch(seed=5)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(cuda_graph=graph, popart_beta=beta, **dict(FLAGS, reward_clipping="none"))
    out = []
    for k in range(steps):
        batch = {key: v.cuda() for key, v in obs_batch(obs, T, B, seed=30 + k).items()}
        if num_tasks:
            batch["reward"] = batch["reward"] * 20.0
            batch["task"] = ((torch.arange(B, device="cuda") + k) % num_tasks).expand(T + 1, B).clone()
        stats = learner.learn(flags, model, actor, batch, tuple(s.clone() for s in model.initial_state(B)), opt, None)
        torch.cuda.synchronize()
        out.append((stats, model.flat_params.clone(),
                    None if num_tasks is None else (model.popart.mu.clone(), model.popart.nu.clone())))
    return out


def test_graphed_learn_is_bit_identical_to_eager():
    eager, graphed = _learn_runs((3, 64, 64), False, 3), _learn_runs((3, 64, 64), True, 3)
    for (se, pe, _), (sg, pg, _) in zip(eager, graphed):
        for key in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
            assert se[key] == sg[key], key
        assert torch.equal(pe, pg)


def test_popart_multitask_x2():
    """K = 4 PopArt learn steps at (3, 64, 64) x2: graphed equals eager bit for bit and the statistics move."""
    eager = _learn_runs((3, 64, 64), False, 3, num_tasks=4, beta=0.1)
    graphed = _learn_runs((3, 64, 64), True, 3, num_tasks=4, beta=0.1)
    for (se, pe, (mue, nue)), (sg, pg, (mug, nug)) in zip(eager, graphed):
        for key in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss", "popart_mu", "popart_sigma"):
            assert se[key] == sg[key], key
        assert torch.equal(pe, pg) and torch.equal(mue, mug) and torch.equal(nue, nug)
        assert np.isfinite(se["total_loss"])
    assert bool((eager[-1][2][0] != 0).any())


@pytest.mark.parametrize("B", [1, 48])
@pytest.mark.parametrize("use_lstm", [False, True])
def test_acting_paths_equal_eager_forward(use_lstm, B):
    from torchbeast_b200 import polybeast_learner
    from torchbeast_b200.acting import GraphedActor, bucket_size
    obs = (3, 64, 64)
    model = make(obs, X2, use_lstm, None)
    model.reset_parameters_like_torch(seed=8)
    model.eval()
    step = obs_batch(obs, 0, B, seed=9)
    real = {k: step[k].cuda() for k in ("frame", "reward", "done")}
    state = tuple(s.cuda() for s in lstm_state(B, use_lstm, seed=10))
    (g_action, g_logits, g_baseline), g_state = GraphedActor(model)(real, state)
    Bk = bucket_size(B)
    pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :1]).expand(-1, Bk - B, *t.shape[2:])], dim=1)
    with torch.no_grad():
        (e_action, e_logits, e_baseline), e_state = model({k: pad(v) for k, v in real.items()}, tuple(pad(s) for s in state))
    assert torch.equal(g_logits, e_logits[:, :B]) and torch.equal(g_baseline, e_baseline[:, :B])
    assert torch.equal(g_action, e_action[:, :B])
    assert all(torch.equal(g, e[:, :B]) for g, e in zip(g_state, e_state))
    with torch.no_grad():
        (x_action, x_logits, x_baseline), x_state = model(real, state)
    got = {}
    batch = mock.Mock()
    batch.get_inputs.return_value = ((step["frame"], step["reward"], step["done"]), tuple(s.cpu() for s in state))
    batch.set_outputs.side_effect = lambda o: got.setdefault("out", o)
    polybeast_learner.inference(types.SimpleNamespace(inference_graph=False), [batch], model)
    (i_action, i_logits, i_baseline), i_state = got["out"]
    assert torch.equal(i_logits, x_logits.cpu()) and torch.equal(i_baseline, x_baseline.cpu())
    assert torch.equal(i_action, x_action.cpu())
    assert all(torch.equal(a, b.cpu()) for a, b in zip(i_state, x_state))


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("obs,channels", [((3, 37, 53), (64, 64, 64)), ((4, 84, 84), (16, 64, 32))])
def test_results_do_not_depend_on_stale_workspace_contents(obs, channels, precision):
    params, batch, state, (w1, w2), _, _ = oracle_case(obs, channels, True)
    model = make(obs, channels, True, precision, params)
    cb = {k: v.cuda() for k, v in batch.items()}
    st = tuple(s.cuda() for s in state)
    runs = []
    for fill in (None, 255, 0):
        if fill is not None:
            model._ws.fill_(fill)
        out = model.learner_forward(cb, st)
        model.learner_backward(w1.float().cuda().contiguous(), w2.float().cuda().contiguous())
        runs.append((out.policy_logits.clone(), out.baseline.clone(), model.flat_grad.clone()))
    for logits, baseline, grads in runs[1:]:
        assert torch.isfinite(grads).all()
        assert torch.equal(logits, runs[0][0]) and torch.equal(baseline, runs[0][1]) and torch.equal(grads, runs[0][2])


def test_shard_rollout_and_state_dict_round_trip():
    from torchbeast_b200 import learner
    obs, T, B = (4, 84, 84), 3, 4
    host = obs_batch(obs, T, B, seed=50)
    model = make(obs, X2, True, None)
    model.reset_parameters_like_torch(seed=3)
    state = tuple(s.cuda() for s in lstm_state(B, True))
    full = model.learner_forward({k: v.cuda() for k, v in host.items()}, state)
    for rank in range(2):
        part, pstate = learner.shard_rollout({k: v.cuda() for k, v in host.items()}, state, rank, 2)
        out = model.learner_forward(part, pstate)
        cols = slice(rank * B // 2, (rank + 1) * B // 2)
        torch.testing.assert_close(out.policy_logits, full.policy_logits[:, cols], rtol=1e-5, atol=1e-5)
    other = make(obs, X2, True, None)
    other.load_state_dict({k: v.cpu() for k, v in model.state_dict().items()})
    assert torch.equal(other.flat_params, model.flat_params)
    again = other.learner_forward({k: v.cuda() for k, v in host.items()}, state)
    assert torch.equal(again.policy_logits, full.policy_logits) and torch.equal(again.baseline, full.baseline)


def test_wide_model_rejects_unstacked_rollouts_and_frame_history():
    from torchbeast_b200 import _lib
    from torchbeast_b200.acting import FrameHistory, GraphedActor
    model = make((4, 84, 84), X2, False, None)
    atari = {k: v.cuda() for k, v in LT.synthetic_batch(2, 2, A, seed=1, with_last_action=False).items()
             if k in ("frame", "reward", "done")}
    with pytest.raises(_lib.TorchBeastB200Error, match=r"unstacked rollouts and newest frames run on the default widths"):
        model.learner_forward(dict(atari, frame=torch.zeros(6, 2, 84, 84, dtype=torch.uint8, device="cuda")))
    model.frame_history = FrameHistory(2)
    step = {k: v[:1] for k, v in atari.items()}
    with pytest.raises(_lib.TorchBeastB200Error, match=r"a frame_history feeds the default widths"):
        model(step)
    with pytest.raises(_lib.TorchBeastB200Error, match=r"a frame_history feeds the default widths"):
        GraphedActor(model)(step)
