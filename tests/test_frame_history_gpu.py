"""GPU: acting on newest frames.  tb_frame_history_fill_u8 against a NumPy FrameStack simulation of many actor streams;
the newest-frame forward of every network backend against the stacked forward on the simulated stacks; graph replays
mixed with eager calls on one history; and graphs of two shapes keeping their own stacked scratch."""
import gc

import numpy as np
import pytest
import torch

from oracle import frames_np as F
from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu

A = 6


@pytest.fixture(autouse=True)
def _collect_graphs():
    """Collect each test's CUDA graphs before the next test can capture one (see tests/test_unstacked_gpu.py)."""
    yield
    gc.collect()
    torch.cuda.synchronize()


class Streams:
    """S environment streams behind atari_wrappers.FrameStack(4), stepped for any subset of them at a time.  A stream's
    stack starts as four zero frames, as a new FrameHistory does, and its first step always starts an episode."""

    def __init__(self, S, seed, done_prob=0.15):
        self.rs = np.random.RandomState(seed)
        self.slots = np.zeros((S, 4, 84, 84), dtype=np.uint8)
        self.started = np.zeros(S, dtype=bool)
        self.done_prob = done_prob

    def step(self, ids, T):
        """T steps of streams `ids` -> (newest frames u8 [T, B, 84, 84], done bool [T, B], stacks u8 [T, B, 4, 84, 84])."""
        ids = np.asarray(ids)
        B = len(ids)
        obs = self.rs.randint(0, 256, size=(T, B, 84, 84)).astype(np.uint8)
        done = self.rs.rand(T, B) < self.done_prob
        done[0] |= ~self.started[ids]
        stacks = np.empty((T, B, 4, 84, 84), dtype=np.uint8)
        for t in range(T):
            for b, s in enumerate(ids):
                if done[t, b]:
                    self.slots[s] = obs[t, b]                       # FrameStack.reset
                else:
                    self.slots[s] = np.concatenate([self.slots[s, 1:], obs[t, b][None]])
                stacks[t, b] = self.slots[s]
        self.started[ids] = True
        return obs, done, stacks

    def history(self):
        """What the device history must hold: channels 1..3 of each stream's latest stack."""
        return self.slots[:, 1:]


def _fill(history, frames, done, ids):
    from torchbeast_b200 import _lib
    T, B = frames.shape[0] - 3, frames.shape[1]
    _lib.check(_lib.lib().tb_frame_history_fill_u8(_lib.ptr(frames), _lib.ptr(done), _lib.ptr(ids), T, B, 84 * 84,
                                                   _lib.ptr(history), history.shape[0], _lib.stream_ptr()),
               "tb_frame_history_fill_u8")


def test_fill_kernel_matches_a_framestack_simulation():
    S = 40
    rs = np.random.RandomState(0)
    sim = Streams(S, seed=1)
    history = torch.zeros(S, 3, 84, 84, dtype=torch.uint8, device="cuda")
    for call in range(30):
        B = int(rs.randint(1, S + 1)) if call else S
        ids = rs.permutation(S)[:B]
        T = int(rs.choice([1, 1, 1, 2, 3, 5]))
        before = sim.history()[ids].copy()
        obs, done, stacks = sim.step(ids, T)
        frames = torch.zeros(T + 3, B, 84, 84, dtype=torch.uint8)
        frames[3:] = torch.from_numpy(obs)
        frames = frames.cuda()
        d = torch.from_numpy(done).cuda()
        _fill(history, frames, d.view(torch.uint8) if call % 2 else d.to(torch.uint8) * 7, torch.from_numpy(ids).cuda())
        got = frames.cpu().numpy()
        assert np.array_equal(got[:3], np.swapaxes(before, 0, 1)), call
        assert np.array_equal(F.restack(got, done), stacks), call
        assert np.array_equal(history.cpu().numpy(), sim.history()), call
    # ids outside [0, S) give zero rows and touch no history; the valid column between them runs as usual
    ids = np.array([S, 5, -1])
    frames = torch.full((4, 3, 84, 84), 9, dtype=torch.uint8)
    frames[3] = torch.from_numpy(np.random.RandomState(2).randint(0, 256, size=(3, 84, 84)).astype(np.uint8))
    frames = frames.cuda()
    want = history.clone()
    want[5] = torch.stack([want[5, 1], want[5, 2], frames[3, 1]])
    before5 = history[5].clone()
    _fill(history, frames, torch.zeros(1, 3, dtype=torch.uint8, device="cuda"), torch.from_numpy(ids).cuda())
    assert not frames[:3, 0].any() and not frames[:3, 2].any()
    assert torch.equal(frames[:3, 1], before5)
    assert torch.equal(history, want)


def _model(net, use_lstm, precision):
    from torchbeast_b200 import nets
    if net == "atari":
        m = nets.AtariNet((4, 84, 84), A, use_lstm, precision=precision)
        m.load_state_dict(LT.random_params(LT.atarinet_param_shapes(A, use_lstm), seed=11))
    else:
        m = nets.ResNet(A, use_lstm, precision=precision)
        m.reset_parameters_like_torch(seed=11)
    return m


def _split(net, out):
    """(action, logits, baseline), state of either network's forward."""
    o, state = out
    if net == "atari":
        return (o["action"], o["policy_logits"], o["baseline"]), tuple(state)
    return tuple(o), tuple(state)


def _step_inputs(model, T, B, seed):
    g = torch.Generator().manual_seed(seed)
    inputs = dict(reward=torch.randn(T, B, generator=g).cuda(),
                  last_action=torch.randint(0, A, (T, B), generator=g).cuda())
    state = tuple((0.1 * torch.randn(s.shape, generator=g)).cuda() for s in model.initial_state(B))
    return inputs, state


def _assert_equal(net, got, want, B=None, padded=False):
    """Columns [:B] of `got` equal those of `want`; `got` has exactly B columns unless it ran `padded`."""
    (ga, gl, gb), gs = _split(net, got)
    (wa, wl, wb), ws = _split(net, want)
    B = B or ga.shape[1]
    assert ga.shape[1] == (wa.shape[1] if padded else B)
    assert torch.equal(gl[:, :B], wl[:, :B]) and torch.equal(gb[:, :B], wb[:, :B]) and torch.equal(ga[:, :B], wa[:, :B])
    assert len(gs) == len(ws) and all(torch.equal(a[:, :B], b[:, :B]) for a, b in zip(gs, ws))


FORWARD_CASES = [(net, lstm, prec, training) for net in ("atari", "resnet") for lstm in (False, True)
                 for prec in ("fp32", "bf16", "bf16x3") for training in (True, False)]


@pytest.mark.parametrize("net,use_lstm,precision,training", FORWARD_CASES)
def test_newest_frame_forward_equals_the_stacked_forward(net, use_lstm, precision, training):
    """20 steps of random stream subsets (T = 3 every fifth step), ids as host, device or default ids; training mode
    runs the autograd forward with a seeded sampler, eval mode the no-grad forward."""
    from torchbeast_b200.acting import FrameHistory
    from torchbeast_b200.sampling import ActionSampler
    S = 6
    model = _model(net, use_lstm, precision)
    model.train(training)
    model.frame_history = FrameHistory(S)
    sim = Streams(S, seed=3, done_prob=0.25)
    rs = np.random.RandomState(4)
    for step in range(20):
        T = 3 if step % 5 == 4 else 1
        kind = step % 3
        B = S if kind == 2 else int(rs.randint(1, S + 1))
        ids = np.arange(B) if kind == 2 else rs.permutation(S)[:B]
        obs, done, stacks = sim.step(ids, T)
        inputs, state = _step_inputs(model, T, B, seed=step)
        inputs["done"] = torch.from_numpy(done).cuda()
        if kind != 2:
            inputs["stream_ids"] = torch.from_numpy(ids) if kind == 0 else torch.from_numpy(ids).cuda()
        outs = []
        for frame in (torch.from_numpy(obs).cuda(), torch.from_numpy(stacks).cuda()):
            if training:
                model.action_sampler = ActionSampler(seed=5, step=step)
            with torch.set_grad_enabled(training):
                outs.append(model(dict(inputs, frame=frame), state))
        _assert_equal(net, outs[0], outs[1])
    assert torch.equal(model.frame_history.buffer.cpu(), torch.from_numpy(sim.history()))


def test_a_newest_frame_without_a_history_is_refused_as_before():
    from torchbeast_b200 import _lib
    model = _model("atari", True, "bf16x3")
    inputs, state = _step_inputs(model, 1, 2, seed=0)
    inputs.update(frame=torch.zeros(1, 2, 84, 84, dtype=torch.uint8, device="cuda"),
                  done=torch.ones(1, 2, dtype=torch.bool, device="cuda"))
    with pytest.raises(_lib.TorchBeastB200Error, match=r"unstacked frame must be uint8 \[T1\+3, B, 84, 84\]"):
        model(inputs, state)


def _pad(t, Bk, value=0):
    out = torch.full((t.shape[0], Bk) + tuple(t.shape[2:]), value, dtype=t.dtype, device=t.device)
    out[:, :t.shape[1]] = t
    return out


def _at_bucket(model, inputs, state, Bk, step):
    """model(inputs, state) on inputs zero-padded to Bk columns (stream ids padded with -1), sampling at `step` of the
    attached sampler's seed; the attached sampler is left as it was."""
    from torchbeast_b200.sampling import ActionSampler
    saved = model.action_sampler
    if saved is not None:
        model.action_sampler = ActionSampler(saved.seed, step)
    padded = {k: _pad(v, Bk) for k, v in inputs.items() if k != "stream_ids"}
    padded["stream_ids"] = _pad(inputs["stream_ids"][None], Bk, -1)[0]
    try:
        with torch.no_grad():
            return model(padded, tuple(_pad(s, Bk) for s in state))
    finally:
        model.action_sampler = saved


@pytest.mark.parametrize("B", [1, 33, 48, 512])
@pytest.mark.parametrize("net", ["atari", "resnet"])
def test_graph_replay_mixed_with_eager_calls(net, B):
    """Six steps on one history, replayed or eager in turn, each equal to the stacked forward at the bucket size.  The
    stream whose id is the first padding column never takes part and keeps its history."""
    from torchbeast_b200.acting import FrameHistory, GraphedActor, bucket_size
    from torchbeast_b200.sampling import ActionSampler
    Bk = bucket_size(B)
    S = Bk + 2
    model = _model(net, True, "bf16x3")
    model.train()
    model.action_sampler = ActionSampler(seed=21)
    model.frame_history = FrameHistory(S)
    sim = Streams(S, seed=B)
    kept = B if Bk > B else None
    if kept is not None:
        model.frame_history.buffer[kept] = 123
        sim.slots[kept, 1:] = 123
    actor = GraphedActor(model)
    rs = np.random.RandomState(B)
    pool = np.array([s for s in range(S) if s != kept])
    for step, mode in enumerate("geggeg"):
        ids = rs.permutation(pool)[:B]
        obs, done, stacks = sim.step(ids, 1)
        inputs, state = _step_inputs(model, 1, B, seed=100 + step)
        inputs.update(done=torch.from_numpy(done).cuda(), stream_ids=torch.from_numpy(ids).cuda())
        at = model.action_sampler.step
        if mode == "g":
            got = actor(dict(inputs, frame=torch.from_numpy(obs).cuda()), state)
        else:
            got = _at_bucket(model, dict(inputs, frame=torch.from_numpy(obs).cuda()), state, Bk, at)
            model.action_sampler.step += 1
        want = _at_bucket(model, dict(inputs, frame=torch.from_numpy(stacks).cuda()), state, Bk, at)
        _assert_equal(net, got, want, B, padded=mode == "e")
        assert model.action_sampler.step == at + 1
    assert actor.captures == 1
    assert torch.equal(model.frame_history.buffer.cpu(), torch.from_numpy(sim.history()))
    if kept is not None:
        assert bool((model.frame_history.buffer[kept] == 123).all())


def test_graphs_hold_their_history_and_key_on_its_size():
    """A graph keeps the history it was captured on alive after the model's history is replaced, so its key's address
    cannot come back as another buffer; a history of another size gets a graph of its own.  A fused backend's graph
    holds no stacked scratch."""
    import weakref
    from torchbeast_b200.acting import FrameHistory, GraphedActor
    B = 3
    model = _model("atari", True, "bf16x3")
    model.eval()
    actor = GraphedActor(model)
    model.frame_history = FrameHistory(4)
    for S, ids in ((4, np.array([2, 0, 3])), (8, np.array([7, 4, 5]))):
        if S == 8:
            held = weakref.ref(model.frame_history.buffer)
            model.frame_history = FrameHistory(S)
            gc.collect()
            assert held() is not None
        sim = Streams(S, seed=S)
        for step in range(3):
            obs, done, stacks = sim.step(ids, 1)
            inputs, state = _step_inputs(model, 1, B, seed=400 + step)
            inputs.update(done=torch.from_numpy(done).cuda(), stream_ids=torch.from_numpy(ids))
            got = actor(dict(inputs, frame=torch.from_numpy(obs).cuda()), state)
            inputs["stream_ids"] = inputs["stream_ids"].cuda()
            _assert_equal("atari", got, _at_bucket(model, dict(inputs, frame=torch.from_numpy(stacks).cuda()), state, 4,
                                                   None), B)
        assert torch.equal(model.frame_history.buffer.cpu(), torch.from_numpy(sim.history()))
    assert actor.captures == 2
    graphs = list(actor._graphs.values())
    assert graphs[0].history is held() and graphs[1].history is model.frame_history.buffer
    assert all(g.scratch is None for g in graphs)


def test_two_shapes_keep_their_own_scratch():
    """ResNet fp32 restacks into the model's stacked scratch, which another shape replaces: graphs at B = 3 and 40,
    with eager forwards of a third shape in between, keep replaying the stacked forward's results."""
    from torchbeast_b200.acting import FrameHistory, GraphedActor, bucket_size
    S = 48
    model = _model("resnet", True, "fp32")
    model.eval()
    model.frame_history = FrameHistory(S)
    sim = Streams(S, seed=7)
    actor = GraphedActor(model)
    rs = np.random.RandomState(8)
    for step, B in enumerate((3, 40, 3, 40)):
        ids = rs.permutation(S)[:B]
        obs, done, stacks = sim.step(ids, 1)
        inputs, state = _step_inputs(model, 1, B, seed=200 + step)
        inputs.update(done=torch.from_numpy(done).cuda(), stream_ids=torch.from_numpy(ids))
        got = actor(dict(inputs, frame=torch.from_numpy(obs).cuda()), state)
        got = ([t.clone() for t in _split("resnet", got)[0]], [s.clone() for s in got[1]])
        # an eager newest-frame forward of another shape replaces the model's scratch (it touches no listed stream)
        other_ids = np.setdiff1d(np.arange(S), ids)[:5]
        o_obs, o_done, _ = sim.step(other_ids, 2)
        o_inputs, o_state = _step_inputs(model, 2, 5, seed=300 + step)
        with torch.no_grad():
            model(dict(o_inputs, frame=torch.from_numpy(o_obs).cuda(), done=torch.from_numpy(o_done).cuda(),
                       stream_ids=torch.from_numpy(other_ids)), o_state)
        inputs["stream_ids"] = inputs["stream_ids"].cuda()
        want = _at_bucket(model, dict(inputs, frame=torch.from_numpy(stacks).cuda()), state, bucket_size(B), None)
        _assert_equal("resnet", ((got[0][0], got[0][1], got[0][2]), got[1]), want, B)
    assert actor.captures == 2
    scratch = [g.scratch for g in actor._graphs.values()]
    assert all(s is not None for s in scratch) and scratch[0].data_ptr() != scratch[1].data_ptr()
    assert torch.equal(model.frame_history.buffer.cpu(), torch.from_numpy(sim.history()))
