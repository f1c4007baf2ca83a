"""IMPALA ResNet on observations other than the Atari stack: Procgen (3, 64, 64), DMLab (3, 72, 96), RGB x 4 (12, 64, 64),
single-channel Atari (1, 84, 84), an odd non-square (3, 37, 53) and the edges of the supported range, on every backend, against the float64 autograd of
oracle/learner_torch.resnet_forward (which reads its sizes from the frame and the parameters), plus the learner, the
graphed paths, PopArt, the acting paths, and the (4, 84, 84) path against the bits it had before the library took an
observation shape."""
import functools
import gc
import types
import unittest.mock as mock

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests import popart_oracle as PO

pytestmark = pytest.mark.gpu

A = 6
# the range's edges: H 17 (last section 3 high), W 33 (last section 5 wide), 126 (the widest row)
SHAPES = [(3, 64, 64), (3, 72, 96), (12, 64, 64), (1, 84, 84), (3, 37, 53), (2, 17, 33), (16, 126, 126), (3, 17, 126),
          (5, 126, 33)]
FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


@pytest.fixture(autouse=True)
def _collect_graphs():
    yield
    gc.collect()
    torch.cuda.synchronize()


def obs_param_shapes(obs, num_actions=A, use_lstm=False):
    """LT.resnet_param_shapes for observations u8 [C, H, W]: first conv (16, C, 3, 3), fc (256, 32 * H_3 * W_3)."""
    from torchbeast_b200.nets import resnet_fc_in
    shapes = LT.resnet_param_shapes(num_actions, use_lstm)
    shapes["feat_convs.0.0.weight"] = (16, obs[0], 3, 3)
    shapes["fc.weight"] = (256, resnet_fc_in(obs))
    return shapes


def obs_batch(obs, T, B, seed):
    batch = LT.synthetic_batch(T, B, A, seed=seed, with_last_action=False)
    rs = np.random.RandomState(seed + 1000)
    batch["frame"] = torch.from_numpy(rs.randint(0, 256, size=(T + 1, B) + tuple(obs)).astype(np.uint8))
    return batch


def make(obs, use_lstm, precision, params=None, **kw):
    from torchbeast_b200 import polybeast_learner
    m = polybeast_learner.Net(A, use_lstm, precision=precision, observation_shape=obs, **kw)
    if params is not None:
        res = m.load_state_dict(params, strict=True)
        assert not res.missing_keys and not res.unexpected_keys
    return m


def lstm_state(B, use_lstm, seed=7):
    if not use_lstm:
        return ()
    rs = np.random.RandomState(seed)
    return tuple(torch.from_numpy(rs.randn(1, B, 256).astype(np.float32) * 0.1) for _ in range(2))


@functools.lru_cache(maxsize=None)
def oracle_case(obs, use_lstm):
    """(params, batch, state, cotangents, float64 outputs, float64 parameter gradients) of a T=2, B=2 case."""
    T, B = 2, 2
    params = LT.random_params(obs_param_shapes(obs, A, use_lstm), seed=sum(obs) + use_lstm)
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
def test_forward_backward_vs_float64_oracle(obs, use_lstm, precision):
    params, batch, state, (w1, w2), (ol, ob), ref = oracle_case(obs, use_lstm)
    model = make(obs, use_lstm, precision, params)
    cb = {k: v.cuda() for k, v in batch.items()}
    out = model.learner_forward(cb, tuple(s.cuda() for s in state))
    logits, baseline = out.policy_logits.cpu().double(), out.baseline.cpu().double()
    assert tuple(logits.shape) == tuple(ol.shape) and tuple(baseline.shape) == tuple(ob.shape)
    if precision == "bf16":   # single-plane bf16 operands and activations: the mixed-precision bounds of test_resnet_gpu.py
        assert rel(logits, ol) < 2e-2 and rel(baseline, ob) < 2e-2
    else:
        np.testing.assert_allclose(logits.numpy(), ol.numpy(), rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(baseline.numpy(), ob.numpy(), rtol=1e-4, atol=1e-4)
    model.learner_backward(w1.float().cuda().contiguous(), w2.float().cuda().contiguous())
    got = {n: p.grad.cpu().double() for n, p in model.named_parameters()}
    assert list(got) == list(ref)
    report = {n: (rel(got[n], ref[n]), float((got[n] * ref[n]).sum() / (got[n].norm() * ref[n].norm()).clamp_min(1e-30)))
              for n in ref}
    if precision == "fp32":
        bad = {n: v for n, v in report.items() if v[0] >= 1e-3}
    elif precision == "bf16x3":
        # the whole gradient within 6e-3; a single tensor can sit further out where a max-pool / ReLU decision flips under
        # the split-bf16 rounding (same per-tensor bounds as test_resnet_gpu.py)
        flat_got = torch.cat([got[n].flatten() for n in ref])
        flat_ref = torch.cat([ref[n].flatten() for n in ref])
        assert rel(flat_got, flat_ref) < 6e-3, report
        bad = {n: v for n, v in report.items() if v[0] >= 3e-2 or v[1] <= 0.9995}
    else:
        # bf16 activations (unit roundoff 2^-9) through 15 convs, 6 frames, random weights.  Measured on an H100 over the
        # first ten of these cases (deterministic run to run): whole gradient 0.013 .. 0.051, median tensor 0.052 .. 0.097, worst tensor
        # 0.36 / cosine 0.944 (resnet2.0.1 at (3, 64, 64) without LSTM, a tensor with a small gradient)
        flat_got = torch.cat([got[n].flatten() for n in ref])
        flat_ref = torch.cat([ref[n].flatten() for n in ref])
        assert rel(flat_got, flat_ref) < 0.1, report
        assert float(np.median([v[0] for v in report.values()])) < 0.15, report
        bad = {n: v for n, v in report.items() if v[0] >= 0.5 or v[1] <= 0.9}
    assert not bad, (bad, report)


def test_default_path_reproduces_the_fixed_geometry_bits():
    """The (4, 84, 84) path with the default widths gives the bits the library gave before it took an observation shape
    (tests/golden/resnet_obs_default_bits.npz, written by tools/make_resnet_default_golden.py with that build): logits,
    baseline, hN and sampled gradients on every backend, from library launches."""
    import importlib.util
    import os
    from tests.common import golden
    from torchbeast_b200 import _lib
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "make_resnet_default_golden.py")
    spec = importlib.util.spec_from_file_location("make_resnet_default_golden", path)
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    g = golden("resnet_obs_default_bits.npz")
    lib = _lib.lib()
    for use_lstm in (False, True):
        for precision in (0, 1, 2):
            before = lib.tb_launch_count()
            got = tool.default_case(use_lstm, precision)
            assert lib.tb_launch_count() > before, (use_lstm, precision)
            for k, v in got.items():
                assert np.array_equal(v, g["%s/lstm%d/p%d" % (k, use_lstm, precision)]), (k, use_lstm, precision)


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
    params = LT.random_params(obs_param_shapes(obs, A, use_lstm), seed=21)
    batch = obs_batch(obs, T, B, seed=22)
    state = lstm_state(B, use_lstm)
    ref = LT.learner_step(params, batch, state, net="resnet", num_actions=A)
    model, actor = make(obs, use_lstm, precision, params), make(obs, use_lstm, precision)
    opt = optim.RMSprop(model, lr=LT.Hyper.learning_rate, momentum=0, eps=LT.Hyper.epsilon, alpha=LT.Hyper.alpha)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 1.0)
    flags = types.SimpleNamespace(unroll_length=T, batch_size=B, learner_device="cuda", **FLAGS)
    stats = {}
    polybeast_learner.learn(flags, queue_of(batch, state), model, actor, opt, sched, stats, mock.Mock())
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(stats[k], float(ref[k]), rtol=1e-4, atol=1e-4, err_msg=k)
    # RMSprop divides by sqrt(v) + eps: an element whose gradient moved by a flipped max-pool / ReLU decision under the
    # split-bf16 rounding moves by up to lr / sqrt(1 - alpha) (same bound as test_resnet_gpu.py)
    patol = 1e-5 if precision == "fp32" else 5e-4
    for n, p in model.named_parameters():
        np.testing.assert_allclose(p.detach().cpu().numpy(), ref["params"][n].numpy(), rtol=1e-4, atol=patol, err_msg=n)
    assert torch.equal(actor.flat_params, model.flat_params)


def _learn_runs(obs, graph, steps, num_tasks=None, T=6, B=4, beta=0.0):
    from torchbeast_b200 import learner, optim
    model = make(obs, True, None, num_tasks=num_tasks)
    actor = make(obs, True, None, num_tasks=num_tasks)
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


def test_popart_multitask_at_dmlab_shape():
    """K = 4 PopArt learn steps at (3, 72, 96): graphed equals eager bit for bit, and one step matches the restatement."""
    eager = _learn_runs((3, 72, 96), False, 3, num_tasks=4, beta=0.1)
    graphed = _learn_runs((3, 72, 96), True, 3, num_tasks=4, beta=0.1)
    for (se, pe, (mue, nue)), (sg, pg, (mug, nug)) in zip(eager, graphed):
        for key in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss", "popart_mu", "popart_sigma"):
            assert se[key] == sg[key], key
        assert torch.equal(pe, pg) and torch.equal(mue, mug) and torch.equal(nue, nug)
    assert bool((eager[-1][2][0] != 0).any())

    from torchbeast_b200 import learner, optim
    obs, T, B, K, beta = (3, 72, 96), 4, 3, 4, 0.1
    batch = obs_batch(obs, T, B, seed=40)
    batch["reward"] = batch["reward"] * 5.0
    task = torch.zeros(T + 1, B, dtype=torch.int64)
    task[:, 0], task[2:, 0], task[:, 1], task[:, 2] = 1, 3, 0, -1
    batch["done"][2, 0] = True
    batch["task"] = task
    shapes = obs_param_shapes(obs, A, False)
    shapes.update({"baseline.weight": (K, 257), "baseline.bias": (K,)})
    p = LT.random_params(shapes, seed=41)
    mu = torch.tensor([0.5, -2.0, 3.0, 10.0], dtype=torch.float64)
    sig = torch.tensor([0.5, 2.0, 5.0, 20.0], dtype=torch.float64)
    nu = sig * sig + mu * mu
    hyper = type("H", (LT.Hyper,), dict(reward_clipping="none"))
    ref = PO.learner_step(p, batch, (), hyper=hyper, net="resnet", num_actions=A, mu=mu, nu=nu, beta=beta, task=task)
    model, actor = make(obs, False, None, num_tasks=K), make(obs, False, None, num_tasks=K)
    model.load_state_dict(dict(p, **{"popart.mu": mu, "popart.nu": nu}))
    opt = optim.RMSprop(model, lr=LT.Hyper.learning_rate, eps=LT.Hyper.epsilon, alpha=LT.Hyper.alpha)
    flags = types.SimpleNamespace(popart_beta=beta, **dict(FLAGS, reward_clipping="none"))
    stats = learner.learn(flags, model, actor, {k: v.cuda() for k, v in batch.items()}, (), opt, None)
    torch.cuda.synchronize()
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(stats[k], float(ref[k]), rtol=2e-4, atol=2e-4, err_msg=k)
    np.testing.assert_allclose(model.popart.mu.cpu().numpy(), ref["mu"].numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(model.popart.nu.cpu().numpy(), ref["nu"].numpy(), rtol=1e-5, atol=1e-6)
    sd = model.state_dict()
    for n in ("baseline.weight", "baseline.bias", "policy.bias", "fc.bias"):
        np.testing.assert_allclose(sd[n].cpu().numpy(), ref["params"][n].numpy(), rtol=1e-3, atol=1e-5, err_msg=n)


@pytest.mark.parametrize("B", [1, 48])
@pytest.mark.parametrize("use_lstm", [False, True])
@pytest.mark.parametrize("obs", [(3, 64, 64), (3, 72, 96)])
def test_acting_paths_equal_eager_forward(obs, use_lstm, B):
    from torchbeast_b200 import polybeast_learner
    from torchbeast_b200.acting import GraphedActor, bucket_size
    model = make(obs, use_lstm, None)
    model.reset_parameters_like_torch(seed=8)
    model.eval()
    step = obs_batch(obs, 0, B, seed=9)
    real = {k: step[k].cuda() for k in ("frame", "reward", "done")}
    state = tuple(s.cuda() for s in lstm_state(B, use_lstm, seed=10))
    # graph replay at the bucket size, against the eager forward on the same zero-padded inputs
    (g_action, g_logits, g_baseline), g_state = GraphedActor(model)(real, state)
    Bk = bucket_size(B)
    pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :1]).expand(-1, Bk - B, *t.shape[2:])], dim=1)
    with torch.no_grad():
        (e_action, e_logits, e_baseline), e_state = model({k: pad(v) for k, v in real.items()}, tuple(pad(s) for s in state))
    assert torch.equal(g_logits, e_logits[:, :B]) and torch.equal(g_baseline, e_baseline[:, :B])
    assert torch.equal(g_action, e_action[:, :B])
    assert all(torch.equal(g, e[:, :B]) for g, e in zip(g_state, e_state))
    # the inference thread body (eager) on one batch of the same inputs
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


def test_acting_rejects_other_shapes_and_frame_history():
    from torchbeast_b200 import _lib, polybeast_learner
    from torchbeast_b200.acting import FrameHistory, GraphedActor
    model = make((3, 64, 64), False, None)
    atari = {k: v.cuda() for k, v in LT.synthetic_batch(0, 2, A, seed=1, with_last_action=False).items()
             if k in ("frame", "reward", "done")}
    with pytest.raises(_lib.TorchBeastB200Error, match=r"GraphedActor takes stacked frames \[1, B, 3, 64, 64\]"):
        GraphedActor(model)(atari)
    batch = mock.Mock()
    batch.get_inputs.return_value = ((atari["frame"].cpu(), atari["reward"].cpu(), atari["done"].cpu()), ())
    with pytest.raises(_lib.TorchBeastB200Error, match=r"inference takes stacked frames \[1, B, 3, 64, 64\]"):
        polybeast_learner.inference(types.SimpleNamespace(inference_graph=False), [batch], model)
    with pytest.raises(_lib.TorchBeastB200Error, match=r"unstacked rollouts and newest frames rebuild \(4, 84, 84\) stacks"):
        model.learner_forward(dict(atari, frame=torch.zeros(4, 2, 84, 84, dtype=torch.uint8, device="cuda")))
    model.frame_history = FrameHistory(2)
    frames = obs_batch((3, 64, 64), 0, 2, seed=2)
    with pytest.raises(_lib.TorchBeastB200Error, match=r"a frame_history rebuilds \(4, 84, 84\) stacks"):
        model({k: frames[k].cuda() for k in ("frame", "reward", "done")})


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("obs", [(3, 37, 53), (12, 64, 64)])
def test_results_do_not_depend_on_stale_workspace_contents(obs, precision):
    params, batch, state, (w1, w2), _, _ = oracle_case(obs, True)
    model = make(obs, True, precision, params)
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


def test_shards_staging_and_sampler_at_new_shape():
    """shard_rollout, a staged batch (staging.spec_for(frame_shape=...)) and the seeded sampler carry the new frame leaf."""
    from torchbeast_b200 import learner, optim, staging
    from torchbeast_b200.sampling import ActionSampler
    obs, T, B = (3, 72, 96), 3, 4
    host = obs_batch(obs, T, B, seed=50)
    spec = staging.spec_for(T, B, A, use_last_action=False, frame_shape=obs)
    assert spec["frame"] == ((T + 1, B) + obs, torch.uint8)
    stager = staging.RolloutStager(spec, torch.device("cuda"))
    stager.put({k: host[k] for k in spec})
    staged, slot = stager.get()
    torch.cuda.synchronize()
    assert torch.equal(staged["frame"].cpu(), host["frame"])
    model = make(obs, True, None)
    model.reset_parameters_like_torch(seed=3)
    state = tuple(s.cuda() for s in lstm_state(B, True))
    full = model.learner_forward({k: staged[k] for k in ("frame", "reward", "done")}, state)
    for rank in range(2):
        part, pstate = learner.shard_rollout({k: v.cuda() for k, v in host.items()}, state, rank, 2)
        assert tuple(part["frame"].shape) == (T + 1, B // 2) + obs
        out = model.learner_forward(part, pstate)
        cols = slice(rank * B // 2, (rank + 1) * B // 2)
        torch.testing.assert_close(out.policy_logits, full.policy_logits[:, cols], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(out.baseline, full.baseline[:, cols], rtol=1e-5, atol=1e-5)
    # seeded sampling in training mode: the same seed and step give the same actions, and they are the sampler's
    # actions for the forward's logits
    model.train()
    inputs = {k: staged[k][:1].contiguous() for k in ("frame", "reward", "done")}
    acts = []
    for _ in range(2):
        model.action_sampler = ActionSampler(17, 3)
        with torch.no_grad():
            (action, logits, _), _ = model(inputs, tuple(s.clone() for s in state))
        acts.append(action)
        assert torch.equal(action, ActionSampler(17, 3).sample(logits))
    assert torch.equal(acts[0], acts[1])
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(**FLAGS)
    stats = learner.learn(flags, model, make(obs, True, None), staged, state, opt, None)
    assert np.isfinite(stats["total_loss"])
    stager.release(slot)
