"""GPU: the replay buffer (torchbeast_b200.replay, tb_replay_mix).  The mix against a torch restatement and the slot
rule of tests/replay_oracle.py, byte for byte; learning with a buffer against learn_step on the batch torch assembles
from the same slots; the graphed learner against the eager one, with the buffer's ring and state compared as well."""
import gc
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests import replay_oracle as RO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)
A = 6
LOSS_KEYS = ("total_loss", "pg_loss", "baseline_loss", "entropy_loss")


@pytest.fixture(autouse=True)
def _collect_graphs():
    yield
    gc.collect()
    torch.cuda.synchronize()


def _batch(T, B, seed, frames="stacked", done_dtype=torch.bool, num_actions=A, obs=(4, 84, 84), num_tasks=None,
           done_prob=0.2):
    b = LT.synthetic_batch(T, B, num_actions, seed=seed, done_prob=done_prob)
    rs = np.random.RandomState(seed + 500)
    if frames == "unstacked":
        b["frame"] = torch.from_numpy(rs.randint(0, 256, size=(T + 4, B, 84, 84)).astype(np.uint8))
    elif tuple(obs) != (4, 84, 84):
        b["frame"] = torch.from_numpy(rs.randint(0, 256, size=(T + 1, B) + tuple(obs)).astype(np.uint8))
    if num_tasks:
        b["task"] = torch.from_numpy(rs.randint(0, num_tasks, size=(T + 1, B)).astype(np.int64))
    b = {k: v.cuda() for k, v in b.items()}
    b["done"] = b["done"].to(done_dtype)
    return b


def _state(layers, B, H, seed):
    g = torch.Generator().manual_seed(seed)
    return tuple((0.1 * torch.randn(layers, B, H, generator=g)).cuda() for _ in range(2))


class Shadow:
    """The ring restated in torch: one [capacity, outer, ...] tensor per leaf, filled as the contract says."""

    def __init__(self, capacity):
        self.capacity, self.rings, self.head, self.size, self.step = capacity, None, 0, 0, 0

    def call(self, leaves, Bf, R, mixing, slots):
        if self.rings is None:
            self.rings = {k: torch.zeros((self.capacity, t.shape[0]) + tuple(t.shape[2:]), dtype=t.dtype, device="cuda")
                          for k, t in leaves.items()}
        mixed = None
        if mixing:
            mixed = {k: torch.cat([t, self.rings[k][slots].transpose(0, 1)], dim=1) for k, t in leaves.items()}
        idx = torch.tensor(RO.overwritten(self.head, self.capacity, Bf), device="cuda")
        for k, t in leaves.items():
            self.rings[k][idx] = t.transpose(0, 1)
        self.head, self.size, self.step = RO.advance(self.head, self.size, self.step, self.capacity, Bf)
        return mixed


def _check_state(buf):
    dev = buf.state.cpu().tolist()
    assert dev == [buf.head, buf.size, buf.seed, buf.step]


@pytest.mark.parametrize("frames,done_dtype", [("stacked", torch.bool), ("unstacked", torch.uint8)])
def test_mix_matches_torch_restatement(frames, done_dtype):
    from torchbeast_b200._lib import TorchBeastB200Error
    from torchbeast_b200.replay import ReplayBuffer
    T, Bf, R, cap, seed = 5, 3, 4, 11, 99
    buf = ReplayBuffer(cap, R, seed=seed, min_size=2, stream_id=5)
    shadow = Shadow(cap)
    for call in range(10):                     # 30 inserts into 11 slots: wraps twice
        batch = _batch(T, Bf, seed=call, frames=frames, done_dtype=done_dtype, num_actions=7, num_tasks=3)
        state = _state(2, Bf, 519, seed=call)
        batch["episode_step"] = torch.zeros(T + 1, Bf, dtype=torch.int32, device="cuda")  # not a learner leaf
        head, size, step = buf.head, buf.size, buf.step
        mixing = RO.mixing(size, cap, Bf, 2)
        out, out_state, fresh = buf.mix(batch, state)
        torch.cuda.synchronize()
        want_slots = RO.slots(R, head, size, cap, Bf, seed, step, 5)
        leaves = {k: batch[k] for k in ("frame", "reward", "done", "policy_logits", "action", "last_action",
                                        "episode_return", "task")}
        leaves.update(h=state[0], c=state[1])
        want = shadow.call(leaves, Bf, R, mixing, torch.from_numpy(want_slots).cuda())
        if mixing:
            assert fresh == Bf
            assert np.array_equal(buf.last_slots.cpu().numpy(), want_slots)
            assert "episode_step" not in out
            got = dict(out, h=out_state[0], c=out_state[1])
            assert sorted(got) == sorted(want)
            for k in want:
                assert got[k].dtype == want[k].dtype and torch.equal(got[k], want[k]), k
        else:
            assert fresh is None and out is batch and all(a is b for a, b in zip(out_state, state))
        _check_state(buf)
        assert (buf.head, buf.size, buf.step) == (shadow.head, shadow.size, shadow.step)
    for ring, k in zip(buf.rings, ("frame", "reward", "done", "policy_logits", "action", "last_action", "episode_return",
                                   "task", "h", "c")):
        assert torch.equal(ring, shadow.rings[k]), k
    with pytest.raises(TorchBeastB200Error, match="columns changed"):
        buf.mix(_batch(T + 1, Bf, seed=0, frames=frames, done_dtype=done_dtype, num_actions=7, num_tasks=3),
                _state(2, Bf, 519, seed=0))


def _atari(precision=None, seed=3):
    from torchbeast_b200 import monobeast
    m = monobeast.AtariNet((4, 84, 84), A, True, precision=precision)
    m.reset_parameters_like_torch(seed=seed)
    return m


def _resnet(seed=3):
    from torchbeast_b200 import polybeast_learner
    m = polybeast_learner.Net(A, True, observation_shape=(3, 64, 64), num_tasks=4)
    m.reset_parameters_like_torch(seed=seed)
    return m


class Learner:
    def __init__(self, make, graph=False, replay=None):
        from torchbeast_b200 import optim
        self.model, self.actor = make(), make()
        self.opt = optim.RMSprop(self.model, lr=0.00048, eps=0.01, alpha=0.99)
        self.flags = types.SimpleNamespace(cuda_graph=graph, **FLAGS)
        if replay is not None:
            self.model.replay = replay

    def learn(self, batch, state):
        from torchbeast_b200 import learner
        stats = learner.learn(self.flags, self.model, self.actor, batch, state, self.opt, None)
        torch.cuda.synchronize()
        return stats

    def learn_step(self, batch, state, fresh=None):
        from torchbeast_b200 import learner
        stats = learner.learn_step(self.flags, self.model, self.actor, batch, state, self.opt, None, fresh_columns=fresh)
        torch.cuda.synchronize()
        return stats


def test_warm_up_is_bit_identical_to_no_buffer():
    from torchbeast_b200.replay import ReplayBuffer
    T, Bf = 4, 4
    plain, buffered = Learner(_atari), Learner(_atari, replay=ReplayBuffer(64, 4, seed=1, min_size=12))
    for k in range(3):
        batch, state = _batch(T, Bf, seed=10 + k), _state(2, Bf, 512 + A + 1, seed=k)
        assert not buffered.model.replay.mixing(Bf)
        sp, sb = plain.learn(batch, state), buffered.learn(batch, state)
        assert sp == sb
        assert torch.equal(plain.model.flat_params, buffered.model.flat_params)
    assert buffered.model.replay.size == 12


CASES = {
    "atari_stacked": (_atari, dict(), (2, 512 + A + 1)),
    "atari_unstacked": (_atari, dict(frames="unstacked"), (2, 512 + A + 1)),
    "resnet_3x64x64_tasks4": (_resnet, dict(obs=(3, 64, 64), num_tasks=4), (1, 256)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_eager_mix_equals_learn_step_on_assembled_batch(case):
    from torchbeast_b200.replay import ReplayBuffer
    make, kw, (layers, H) = CASES[case]
    T, Bf, R, cap = 4, 4, 4, 10
    mixed_run = Learner(make, replay=ReplayBuffer(cap, R, seed=21, min_size=4))
    ref = Learner(make)
    shadow = Shadow(cap)
    buf = mixed_run.model.replay
    for k in range(3):                          # one warm-up step, two mixing steps
        batch, state = _batch(T, Bf, seed=40 + k, **kw), _state(layers, Bf, H, seed=k)
        mixing = buf.mixing(Bf)
        assert mixing == (k > 0)
        stats = mixed_run.learn(batch, state)
        leaves = {key: v for key, v in batch.items()
                  if key in ("frame", "reward", "done", "policy_logits", "action", "last_action", "episode_return", "task")}
        leaves.update(h=state[0], c=state[1])
        slots = buf.last_slots if mixing else None
        want = shadow.call(leaves, Bf, R, mixing, slots)
        if mixing:
            mb = {key: v for key, v in want.items() if key not in ("h", "c")}
            ref_stats = ref.learn_step(mb, (want["h"], want["c"]), fresh=Bf)
        else:
            ref_stats = ref.learn_step(batch, state)
        for key in LOSS_KEYS:
            assert stats[key] == ref_stats[key], (k, key)
        assert stats["episode_returns"] == ref_stats["episode_returns"]
        assert torch.equal(mixed_run.model.flat_params, ref.model.flat_params), k
        if getattr(ref.model, "popart", None) is not None:
            assert torch.equal(mixed_run.model.popart.mu, ref.model.popart.mu)


def _ring_copy(buf):
    return [r.clone() for r in buf.rings], buf.state.clone(), (buf.head, buf.size, buf.seed, buf.step)


def _assert_same_buffer(a, b):
    ra, sa, ma = a
    rb, sb, mb = b
    assert ma == mb
    assert torch.equal(sa, sb)
    assert all(torch.equal(x, y) for x, y in zip(ra, rb))


def test_graphed_equals_eager_across_warm_up():
    from torchbeast_b200.replay import ReplayBuffer
    T, Bf, R, cap = 4, 4, 4, 14
    runs = {g: Learner(_atari, graph=g, replay=ReplayBuffer(cap, R, seed=8, min_size=8)) for g in (False, True)}
    for k in range(8):                          # warm-up for 2 steps, then mixing; the ring is full from step 4
        batch, state = _batch(T, Bf, seed=60 + k), _state(2, Bf, 512 + A + 1, seed=k)
        mixing = runs[True].model.replay.mixing(Bf)
        assert mixing == (k >= 2)
        se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
        for key in LOSS_KEYS:
            assert se[key] == sg[key], (k, key)
        assert se["episode_returns"] == sg["episode_returns"]
        assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params), k
        _assert_same_buffer(_ring_copy(runs[False].model.replay), _ring_copy(runs[True].model.replay))
        _check_state(runs[True].model.replay)
        if mixing:
            assert torch.equal(runs[False].model.replay.last_slots, runs[True].model.replay.last_slots)
    assert len(runs[True].model._tb_graphs) == 2     # one graph per phase


@pytest.mark.parametrize("fill_calls", [1, 3])
def test_capture_leaves_the_buffer_untouched(fill_calls):
    from torchbeast_b200 import learner
    from torchbeast_b200.replay import ReplayBuffer
    T, Bf, R, cap = 4, 4, 4, 10
    run = Learner(_atari, graph=True, replay=ReplayBuffer(cap, R, seed=2, min_size=4))
    buf = run.model.replay
    for k in range(fill_calls):                 # 3 calls fill the 10 slots
        buf.mix(_batch(T, Bf, seed=80 + k), _state(2, Bf, 512 + A + 1, seed=k))
    torch.cuda.synchronize()
    assert buf.size == min(fill_calls * Bf, cap)
    before = _ring_copy(buf)
    params = run.model.flat_params.clone()
    learner.GraphedLearner(run.flags, run.model, run.actor, run.opt, _batch(T, Bf, seed=90),
                           _state(2, Bf, 512 + A + 1, seed=9))
    torch.cuda.synchronize()
    _assert_same_buffer(before, _ring_copy(buf))
    assert torch.equal(params, run.model.flat_params)


@pytest.mark.parametrize("graph", [False, True])
def test_episode_returns_come_from_fresh_columns_only(graph):
    from torchbeast_b200.replay import ReplayBuffer
    T, Bf = 4, 4
    run = Learner(_atari, graph=graph, replay=ReplayBuffer(12, 4, seed=4, min_size=4))
    with_done = _batch(T, Bf, seed=1)
    with_done["done"][:] = True
    stats = run.learn(with_done, _state(2, Bf, 512 + A + 1, seed=1))       # warm-up: counted, the columns are fresh
    assert len(stats["episode_returns"]) == T * Bf
    no_done = _batch(T, Bf, seed=2)
    no_done["done"][:] = False
    assert run.model.replay.mixing(Bf)
    stats = run.learn(no_done, _state(2, Bf, 512 + A + 1, seed=2))          # every done is in a replayed column
    assert stats["episode_returns"] == ()


def test_host_batch_and_polybeast_queue_match_device_path():
    from torchbeast_b200 import polybeast_learner
    from torchbeast_b200.replay import ReplayBuffer
    T, Bf = 4, 4
    mk = lambda: ReplayBuffer(10, 4, seed=6, min_size=4)   # noqa: E731
    dev_run, host_run, poly_run = Learner(_atari, replay=mk()), Learner(_atari, replay=mk()), Learner(_atari, replay=mk())
    batches = []
    for k in range(3):
        b = _batch(T, Bf, seed=70 + k)
        del b["last_action"]                       # the polybeast nest has none: learn() uses `action`
        batches.append((b, _state(2, Bf, 512 + A + 1, seed=k)))
    for b, s in batches:
        dev_run.learn(b, s)
        host_run.learn({k: v.cpu() for k, v in b.items()}, tuple(x.cpu() for x in s))
    assert torch.equal(dev_run.model.flat_params, host_run.model.flat_params)

    class Queue(list):
        def size(self):
            return 0

    queue = Queue()
    for b, s in batches:
        env = (b["frame"].cpu(), b["reward"].cpu(), b["done"].cpu(), b["episode_step"].cpu(), b["episode_return"].cpu())
        agent = (b["action"].cpu(), b["policy_logits"].cpu(), b["baseline"].cpu())
        queue.append(((env, agent), tuple(x.cpu() for x in s)))
    poly_run.flags.unroll_length, poly_run.flags.batch_size = T, Bf
    polybeast_learner.learn(poly_run.flags, queue, poly_run.model, poly_run.actor, poly_run.opt, None, {},
                            types.SimpleNamespace(log=lambda stats: None))
    torch.cuda.synchronize()
    assert torch.equal(dev_run.model.flat_params, poly_run.model.flat_params)
    _assert_same_buffer(_ring_copy(dev_run.model.replay), _ring_copy(poly_run.model.replay))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_keep_identical_replicas():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29547", os.path.join(ROOT, "tools", "replay_dp_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
    assert line["replicas_bit_identical"] is True and line["slots_differ"] is True, line
