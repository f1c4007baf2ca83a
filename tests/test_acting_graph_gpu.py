"""GPU: the T=1 acting forward replayed as a CUDA graph (torchbeast_b200.acting.GraphedActor) against the eager forward at
the bucket size on the same padded inputs and against the torch oracle; the sampler's step sequence; weights changed
between replays; graphs keeping their own buffers; no library launch per replay; polybeast's inference thread with the
graph; and the learner's graphs keeping their workspaces across batch shapes."""
import threading
import types
import unittest.mock as mock

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu

A = 6


def _net(kind, use_lstm, seed):
    from torchbeast_b200 import monobeast, polybeast_learner
    if kind == "atari":
        model = monobeast.AtariNet((4, 84, 84), A, use_lstm)
        params = LT.random_params(LT.atarinet_param_shapes(A, use_lstm), seed=seed)
    else:
        model = polybeast_learner.Net(A, use_lstm)
        params = LT.random_params(LT.resnet_param_shapes(A, use_lstm), seed=seed)
    model.load_state_dict(params)
    return model, params


def _inputs(model, B, seed):
    """One [1, B] acting step (CUDA) and a random core state."""
    batch = LT.synthetic_batch(0, B, A, seed=seed, with_last_action=getattr(model, "needs_last_action", False))
    names = ("frame", "reward", "done", "last_action") if getattr(model, "needs_last_action", False) \
        else ("frame", "reward", "done")
    inputs = {k: batch[k].cuda() for k in names}
    g = torch.Generator().manual_seed(seed)
    state = tuple((0.1 * torch.randn(s.shape, generator=g)).cuda() for s in model.initial_state(B))
    return inputs, state


def _pad(t, Bk):
    out = torch.zeros((t.shape[0], Bk) + tuple(t.shape[2:]), dtype=t.dtype, device=t.device)
    out[:, :t.shape[1]] = t
    return out


def _split(kind, outputs):
    """(action, logits, baseline), state of either network's forward."""
    out, state = outputs
    if kind == "atari":
        return (out["action"], out["policy_logits"], out["baseline"]), tuple(state)
    return tuple(out), tuple(state)


def _eager_at_bucket(model, inputs, state, step=None):
    """The eager forward at the bucket size on the zero-padded inputs, sampling at `step` of the attached sampler's seed
    (the attached sampler itself is left as it was)."""
    from torchbeast_b200.acting import bucket_size
    from torchbeast_b200.sampling import ActionSampler
    B = inputs["frame"].shape[1]
    Bk = bucket_size(B)
    saved = model.action_sampler
    if saved is not None:
        model.action_sampler = ActionSampler(saved.seed, step)
    try:
        with torch.no_grad():
            return model({k: _pad(v, Bk) for k, v in inputs.items()}, tuple(_pad(s, Bk) for s in state))
    finally:
        model.action_sampler = saved


def _assert_real_rows_equal(kind, graphed, eager, B):
    (ga, gl, gb), gs = _split(kind, graphed)
    (ea, el, eb), es = _split(kind, eager)
    assert ga.shape[1] == B and gl.shape[1] == B and gb.shape[1] == B
    assert torch.equal(gl, el[:, :B]) and torch.equal(gb, eb[:, :B]) and torch.equal(ga, ea[:, :B])
    assert len(gs) == len(es)
    for a, b in zip(gs, es):
        assert a.shape[1] == B and torch.equal(a, b[:, :B])


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("B", [1, 33, 48, 512])
@pytest.mark.parametrize("use_lstm", [False, True])
@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_graphed_forward_equals_eager_and_oracle(kind, use_lstm, B, training):
    from torchbeast_b200.acting import GraphedActor
    from torchbeast_b200.sampling import ActionSampler
    model, params = _net(kind, use_lstm, seed=11)
    model.train(training)
    if training:
        model.action_sampler = ActionSampler(seed=77, step=1000)
    inputs, state = _inputs(model, B, seed=B)
    actor = GraphedActor(model)
    graphed = actor(inputs, state)
    if training:
        assert model.action_sampler.step == 1001
    _assert_real_rows_equal(kind, graphed, _eager_at_bucket(model, inputs, state, step=1000), B)
    (action, logits, baseline), new_state = _split(kind, graphed)
    if not training:
        assert torch.equal(action, logits.argmax(-1))
    cpu = {k: v.cpu() for k, v in inputs.items()}
    cstate = tuple(s.cpu() for s in state)
    if kind == "atari":
        ol, ob, ostate = LT.atarinet_forward(params, cpu["frame"], cpu["reward"], cpu["done"], cpu["last_action"], cstate)
    else:
        ol, ob, ostate = LT.resnet_forward(params, cpu["frame"], cpu["reward"], cpu["done"], cstate)
    np.testing.assert_allclose(logits.cpu().numpy(), ol.numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(baseline.cpu().numpy(), ob.numpy(), rtol=1e-4, atol=1e-4)
    for a, b in zip(new_state, ostate):
        np.testing.assert_allclose(a.cpu().numpy(), b.numpy(), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_step_sequence_and_sampler_swap(kind):
    """Five graphed calls (state carried) == five eager calls with a fresh sampler at the same seed, mixing the two
    changes nothing, and a sampler swapped in between calls takes effect without a new capture.  B is a power of two,
    so the eager calls run at the graph's own size."""
    from torchbeast_b200.acting import GraphedActor
    from torchbeast_b200.sampling import ActionSampler
    B = 16
    model, _ = _net(kind, True, seed=21)
    model.train()
    steps = [_inputs(model, B, seed=100 + t)[0] for t in range(5)]

    def run(mode):
        model.action_sampler = ActionSampler(seed=5)
        actor = GraphedActor(model)
        state, actions = model.initial_state(B), []
        for t, inputs in enumerate(steps):
            if mode == "graphed" or (mode == "mixed" and t % 2):
                out = actor(inputs, state)
            else:
                with torch.no_grad():
                    out = model(inputs, state)
            (a, _, _), st = _split(kind, out)
            actions.append(a.clone())
            state = tuple(s.clone() for s in st)
        return actions, actor

    graphed, actor = run("graphed")
    assert model.action_sampler.step == 5 and actor.captures == 1
    eager, _ = run("eager")
    mixed, _ = run("mixed")
    for g, e, m in zip(graphed, eager, mixed):
        assert torch.equal(g, e) and torch.equal(m, e)
    # swap in another sampler: the next replay samples at ITS seed and step
    state = model.initial_state(B)
    model.action_sampler = ActionSampler(seed=9, step=40)
    out = actor(steps[0], state)
    assert actor.captures == 1 and model.action_sampler.step == 41
    want = _eager_at_bucket(model, steps[0], state, step=40)
    _assert_real_rows_equal(kind, out, want, B)


def test_weights_changed_between_replays_and_moved_weights():
    from torchbeast_b200.acting import GraphedActor
    B = 8
    model, _ = _net("atari", True, seed=31)
    model.eval()
    inputs, state = _inputs(model, B, seed=32)
    actor = GraphedActor(model)
    first = _split("atari", actor(inputs, state))[0][1].clone()
    other, _ = _net("atari", True, seed=33)
    model.copy_params_from(other)
    out = actor(inputs, state)
    assert not torch.equal(_split("atari", out)[0][1], first)
    _assert_real_rows_equal("atari", out, _eager_at_bucket(model, inputs, state), B)
    model.load_state_dict(LT.random_params(LT.atarinet_param_shapes(A, True), seed=34))  # key by key
    _assert_real_rows_equal("atari", actor(inputs, state), _eager_at_bucket(model, inputs, state), B)
    assert actor.captures == 1
    old = model.flat_params  # held, so the moved buffer cannot come back at the same address
    model.cpu()
    model.cuda()
    assert model.flat_params.data_ptr() != old.data_ptr()
    out = actor(inputs, state)
    assert actor.captures == 2
    _assert_real_rows_equal("atari", out, _eager_at_bucket(model, inputs, state), B)


def test_graphs_keep_their_buffers():
    """B = 1, 48, 512, 48, 1 on one model, with eager forwards at B = 7 in between that replace the model's workspace."""
    from torchbeast_b200.acting import GraphedActor
    from torchbeast_b200.sampling import ActionSampler
    model, _ = _net("atari", True, seed=41)
    model.train()
    model.action_sampler = ActionSampler(seed=42)
    actor = GraphedActor(model)
    other, other_state = _inputs(model, 7, seed=43)
    for i, B in enumerate((1, 48, 512, 48, 1)):
        inputs, state = _inputs(model, B, seed=50 + i)
        step = model.action_sampler.step
        out = actor(inputs, state)
        got = ([t.clone() for t in _split("atari", out)[0]], [s.clone() for s in out[1]])
        with torch.no_grad():
            model(other, other_state)
        want = _eager_at_bucket(model, inputs, state, step=step)
        _assert_real_rows_equal("atari", (dict(action=got[0][0], policy_logits=got[0][1], baseline=got[0][2]), got[1]),
                                want, B)
        with torch.no_grad():
            model(other, other_state)
    assert actor.captures == 3


def test_replay_adds_no_library_launch():
    from torchbeast_b200 import _lib
    from torchbeast_b200.acting import GraphedActor
    from torchbeast_b200.sampling import ActionSampler
    model, _ = _net("atari", True, seed=51)
    model.train()
    model.action_sampler = ActionSampler(seed=1)
    inputs, state = _inputs(model, 48, seed=52)
    actor = GraphedActor(model)
    actor(inputs, state)  # capture
    torch.cuda.synchronize()
    n0 = _lib.lib().tb_launch_count()
    for _ in range(3):
        actor(inputs, state)
    torch.cuda.synchronize()
    assert _lib.lib().tb_launch_count() == n0


def _mock_batcher(model, sizes, seed):
    """DynamicBatcher stand-in: one batch per size, with CPU leaves like the reference's."""
    mbs = []
    for i, B in enumerate(sizes):
        batch = LT.synthetic_batch(0, B, A, seed=seed + i)
        env = tuple(batch[k] for k in ("frame", "reward", "done", "episode_step", "episode_return", "last_action"))
        g = torch.Generator().manual_seed(seed + i)
        state = tuple(0.1 * torch.randn(s.shape, generator=g) for s in model.initial_state(B))
        mb = mock.MagicMock()
        mb.get_inputs = mock.Mock(return_value=(env, state))
        mbs.append(mb)
    batcher = mock.MagicMock()
    batcher.__iter__.return_value = iter(mbs)
    return batcher, mbs


def _outputs_of(mb):
    (outputs,), kw = mb.set_outputs.call_args
    assert kw == {}
    (action, logits, baseline), state = outputs
    for t in (action, logits, baseline) + tuple(state):
        assert t.device == torch.device("cpu")
    return action, logits, baseline, tuple(state)


@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_inference_with_the_graph_gives_the_eager_outputs(kind):
    """B = 48 runs at its bucket, 64, where a GEMM's split-K partition may differ from B = 48's: the floats agree to
    rounding, the actions exactly."""
    from torchbeast_b200 import polybeast_learner
    from torchbeast_b200.sampling import ActionSampler
    model, _ = _net(kind, True, seed=61)
    model.train()
    results = []
    for graph in (False, True):
        model.action_sampler = ActionSampler(seed=3)
        batcher, mbs = _mock_batcher(model, (48, 3), seed=62)
        polybeast_learner.inference(types.SimpleNamespace(actor_device="cuda:0", inference_graph=graph), batcher, model)
        assert model.action_sampler.step == 2
        results.append([_outputs_of(mb) for mb in mbs])
    assert "_tb_graphed_actor" in model.__dict__
    for eager, graphed in zip(*results):
        assert torch.equal(eager[0], graphed[0])
        for e, g in zip(eager[1:3] + eager[3], graphed[1:3] + graphed[3]):
            assert e.shape == g.shape
            np.testing.assert_allclose(g.numpy(), e.numpy(), rtol=1e-5, atol=1e-6)


def test_two_inference_threads_each_get_their_own_outputs():
    """Two graphed inference threads share one model, one lock and (B = 40 and 48 are both bucket 64) one graph."""
    from torchbeast_b200 import polybeast_learner
    model, _ = _net("atari", True, seed=71)
    model.eval()
    lock = threading.Lock()
    flags = types.SimpleNamespace(actor_device="cuda:0", inference_graph=True)
    work = [_mock_batcher(model, (40,) * 6, seed=100), _mock_batcher(model, (48,) * 6, seed=200)]
    errors = []

    def body(batcher):
        try:
            torch.cuda.set_device(0)
            polybeast_learner.inference(flags, batcher, model, lock)
        except Exception as e:  # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=body, args=(b,)) for b, _ in work]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert model._tb_graphed_actor.captures == 1
    for _, mbs in work:
        for mb in mbs:
            action, logits, baseline, state = _outputs_of(mb)
            env, st = mb.get_inputs.return_value
            inputs = dict(frame=env[0].cuda(), reward=env[1].cuda(), done=env[2].cuda(), last_action=env[5].cuda())
            with torch.no_grad():
                out, want_state = model(inputs, tuple(s.cuda() for s in st))
            np.testing.assert_allclose(logits.numpy(), out["policy_logits"].cpu().numpy(), rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(baseline.numpy(), out["baseline"].cpu().numpy(), rtol=1e-5, atol=1e-6)
            assert torch.equal(action, logits.argmax(-1))
            for a, b in zip(state, want_state):
                np.testing.assert_allclose(a.numpy(), b.cpu().numpy(), rtol=1e-5, atol=1e-6)


def test_learner_graphs_keep_their_workspaces():
    """learn() with cuda_graph over two alternating batch shapes, with an eager forward of a third shape in between,
    equals eager learn_step step for step."""
    from torchbeast_b200 import learner, monobeast, optim
    params = LT.random_params(LT.atarinet_param_shapes(A, True), seed=81)
    runs = []
    for graph in (False, True):
        model = monobeast.AtariNet((4, 84, 84), A, True)
        actor = monobeast.AtariNet((4, 84, 84), A, True)
        model.load_state_dict(params)
        actor.load_state_dict(params)
        opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
        flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5,
                                      entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=graph)
        third = {k: v.cuda() for k, v in LT.synthetic_batch(2, 5, A, seed=82).items()}
        out = []
        for step in range(6):
            T, B = ((4, 2), (6, 3))[step % 2]
            batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=90 + step).items()}
            state = model.initial_state(B)
            if graph:
                s = learner.learn(flags, model, actor, batch, state, opt, None)
            else:
                s = learner.learn_step(flags, model, actor, batch, state, opt, None)
            model.learner_forward(third, model.initial_state(5))
            out.append((s["total_loss"], s["pg_loss"], model.flat_params.clone()))
        runs.append(out)
    for (le, pe, we), (lg, pg, wg) in zip(*runs):
        assert le == lg and pe == pg and torch.equal(we, wg)
