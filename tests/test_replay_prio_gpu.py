"""GPU: prioritised replay.  The sampler against the NumPy rule of tests/replay_prio_oracle.py; the weighted loss
against the unweighted kernel and a float64 restatement; the priority update against NumPy; learning with a
prioritised buffer against learn_step on the batch the torch Shadow ring assembles, eager and graphed."""
import types

import numpy as np
import pytest
import torch

from tests import replay_oracle as RO
from tests import replay_prio_oracle as PO
from tests.test_replay_gpu import (A, FLAGS, LOSS_KEYS, Learner, Shadow, _atari, _batch, _collect_graphs,  # noqa: F401
                                   _state)

pytestmark = pytest.mark.gpu
KEYS = ("frame", "reward", "done", "policy_logits", "action", "last_action", "episode_return", "task")


def _resnet(seed=3):
    from torchbeast_b200 import polybeast_learner
    m = polybeast_learner.Net(A, True, observation_shape=(3, 64, 64))
    m.reset_parameters_like_torch(seed=seed)
    return m


def _prio_buffer(cap, R, seed, min_size, alpha=0.6, beta=0.4):
    from torchbeast_b200.replay import ReplayBuffer
    return ReplayBuffer(cap, R, seed=seed, min_size=min_size, priority_exponent=alpha, importance_exponent=beta)


def _sample(pr, head, size, cap, Bf, R, seed, step, sid, alpha, beta, eps):
    from torchbeast_b200 import _lib
    p = _lib.ptr
    prio = torch.tensor([alpha, beta, 0.9, eps], dtype=torch.float64, device="cuda")
    hs = torch.tensor([head, size], dtype=torch.int64, device="cuda")
    ss = torch.tensor([seed, step], dtype=torch.int64, device="cuda")
    slots = torch.full((Bf + R,), -7, dtype=torch.int64, device="cuda")
    w = torch.full((Bf + R,), -1.0, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().tb_replay_sample_prioritized(p(pr), p(prio), p(hs), p(ss), Bf, R, cap, sid, p(slots), p(w),
                                                       _lib.stream_ptr()), "tb_replay_sample_prioritized")
    torch.cuda.synchronize()
    return slots.cpu().numpy(), w.cpu().numpy()


@pytest.mark.parametrize("alpha", [1.0, 0.6])
@pytest.mark.parametrize("cap,Bf,R,head,size", [(40, 8, 64, 5, 40), (700, 8, 256, 3, 700), (700, 8, 256, 100, 350),
                                                (5000, 16, 512, 4321, 5000), (70000, 32, 300, 12, 70000)])
def test_sampler_matches_oracle(alpha, cap, Bf, R, head, size):
    rs = np.random.RandomState(cap)
    pr_np = rs.gamma(0.5, size=cap).astype(np.float32)
    pr_np[rs.rand(cap) < 0.05] = 0.0
    pr = torch.from_numpy(pr_np).cuda()
    boundary = 0
    for step in range(3):
        slots, w = _sample(pr, head, size, cap, Bf, R, 77, step, 3, alpha, 0.4, 1e-6)
        again = _sample(pr, head, size, cap, Bf, R, 77, step, 3, alpha, 0.4, 1e-6)
        assert np.array_equal(slots, again[0]) and np.array_equal(w.view(np.int32), again[1].view(np.int32))
        assert np.array_equal(slots[:Bf], (head + np.arange(Bf)) % cap) and np.all(w[:Bf] == 1.0)
        want, want_w, margin = PO.prioritized(pr_np, R, head, size, cap, Bf, 77, step, 3, alpha, 0.4, 1e-6)
        if alpha == 1.0:
            assert np.array_equal(slots[Bf:], want)
        else:
            near = margin < 1e-12
            boundary += int(near.sum())
            assert np.array_equal(slots[Bf:][~near], want[~near])
        same = slots[Bf:] == want
        np.testing.assert_allclose(w[Bf:][same], want_w[same], rtol=1e-6)
        assert np.all(w[Bf:] > 0) and np.all(w[Bf:] <= 1)
    assert boundary == 0


def test_sampler_without_draws_writes_fresh_slots_only():
    pr = torch.zeros(10, device="cuda")
    slots, w = _sample(pr, 8, 0, 10, 4, 0, 1, 0, 0, 0.6, 0.4, 1e-6)
    assert slots.tolist() == [8, 9, 0, 1] and w.tolist() == [1.0] * 4


def _loss_inputs(T, B, seed):
    rs = np.random.RandomState(seed)
    cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
    return dict(behavior_policy_logits=cu(rs.randn(T, B, A).astype(np.float32)),
                target_policy_logits=cu(rs.randn(T, B, A).astype(np.float32)),
                actions=cu(rs.randint(0, A, size=(T, B)).astype(np.int64)),
                rewards=cu((2 * rs.randn(T, B)).astype(np.float32)), done=cu(rs.rand(T, B) < 0.1),
                values=cu(rs.randn(T, B).astype(np.float32)), bootstrap_value=cu(rs.randn(B).astype(np.float32)))


def _hp_block():
    from torchbeast_b200 import learner
    block = torch.zeros(learner.HPARAMS.itemsize, dtype=torch.uint8, device="cuda")
    flags = types.SimpleNamespace(**FLAGS)
    learner.publish_hparams(learner.pack_hparams(flags), block)
    return block


def _bits_equal(a, b):
    return all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b) if x is not None)


@pytest.mark.parametrize("T,B", [(80, 32), (5, 70), (300, 8)])
def test_weighted_loss_with_unit_weights_is_bit_identical(T, B):
    from torchbeast_b200 import learner
    kw = _loss_inputs(T, B, T + B)
    ones = torch.ones(B, device="cuda")
    costs = dict(discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006)
    hp = _hp_block()
    for hparams_dev in (None, hp):
        plain = learner.impala_loss_fwd_bwd(**kw, **costs, hparams_dev=hparams_dev)
        weighted = learner.impala_loss_fwd_bwd(**kw, **costs, hparams_dev=hparams_dev, column_weights=ones)
        torch.cuda.synchronize()
        assert _bits_equal(plain, weighted)


@pytest.mark.parametrize("T,B", [(80, 32), (5, 70)])
def test_weighted_loss_matches_float64_restatement(T, B):
    from torchbeast_b200 import learner
    kw = _loss_inputs(T, B, 3 * T + B)
    g = torch.Generator().manual_seed(B)
    w = torch.rand(B, generator=g).cuda()
    w[3] = 0.0
    bc, ec = 0.5, 0.0006
    plain = learner.impala_loss_fwd_bwd(**kw, baseline_cost=bc, entropy_cost=ec)
    out = learner.impala_loss_fwd_bwd(**kw, baseline_cost=bc, entropy_cost=ec, column_weights=w,
                                      hparams_dev=_hp_block())
    torch.cuda.synchronize()
    # the terms are weighted after they are formed: the gradients are the unweighted ones times w, to the bit
    assert torch.equal(out.grad_logits[:T], plain.grad_logits[:T] * w[None, :, None])
    assert torch.equal(out.grad_values[:T], plain.grad_values[:T] * w[None, :])
    assert torch.all(out.grad_logits[:, 3] == 0) and torch.all(out.grad_values[:, 3] == 0)
    assert torch.all(out.grad_logits[T] == 0) and torch.all(out.grad_values[T] == 0)
    for a, b in zip(out[:5], plain[:5]):
        assert torch.equal(a, b)                      # vs, pg_adv, log_rhos, log-probabilities are not weighted
    # losses in float64 from the kernel's own per-row quantities
    d = torch.float64
    wd = w.to(d)[None, :]
    logp = torch.log_softmax(kw["target_policy_logits"].to(d), dim=-1)
    pg = (-out.target_action_log_probs.to(d) * out.pg_advantages.to(d) * wd).sum()
    bl = bc * (0.5 * (out.vs.to(d) - kw["values"].to(d)) ** 2 * wd).sum()
    en = ec * ((logp.exp() * logp).sum(-1) * wd).sum()
    want = torch.stack([pg, bl, en, pg + bl + en]).cpu()
    np.testing.assert_allclose(out.losses.cpu().double().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)
    # and the gradients against float64 autograd
    tl = kw["target_policy_logits"].to(d).requires_grad_()
    v = kw["values"].to(d).requires_grad_()
    lp = torch.log_softmax(tl, dim=-1)
    lpa = lp.gather(-1, kw["actions"][..., None])[..., 0]
    total = ((-lpa * out.pg_advantages.to(d) + bc * 0.5 * (out.vs.to(d) - v) ** 2 + ec * (lp.exp() * lp).sum(-1))
             * wd).sum()
    total.backward()
    np.testing.assert_allclose(out.grad_logits[:T].cpu().numpy(), tl.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(out.grad_values[:T].cpu().numpy(), v.grad.cpu().numpy(), rtol=1e-4, atol=1e-5)


def test_priority_update_matches_numpy():
    from torchbeast_b200 import _lib
    T, Bf, R, cap, eta = 80, 16, 16, 200, 0.9
    rs = np.random.RandomState(5)
    vs, values = rs.randn(T, Bf + R).astype(np.float32), rs.randn(T, Bf + R).astype(np.float32)
    values[7, 2] = np.nan
    vs[3, 20] = np.inf
    slots = np.concatenate([(190 + np.arange(Bf)) % cap, rs.choice(np.arange(20, 60), R)]).astype(np.int64)
    slots[Bf + 3] = slots[Bf + 9] = slots[Bf + 15] = 44                      # drawn three times: column Bf+15 wins
    before = rs.rand(cap).astype(np.float32)
    pr = torch.from_numpy(before).cuda()
    prio = torch.tensor([0.6, 0.4, eta, 1e-6], dtype=torch.float64, device="cuda")
    p = _lib.ptr
    dvs, dvalues, dslots = (torch.from_numpy(x).cuda() for x in (vs, values, slots))   # alive until the kernel ran
    _lib.check(_lib.lib().tb_replay_update_priorities(p(dvs), p(dvalues), T, Bf + R, p(dslots), p(prio), p(pr),
                                                      _lib.stream_ptr()), "tb_replay_update_priorities")
    torch.cuda.synchronize()
    got = pr.cpu().numpy()
    want = PO.priority_update(vs, values, slots, eta, before)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert got[slots[2]] == 0.0 and got[slots[20]] == 0.0
    untouched = sorted(set(range(cap)) - set(slots.tolist()))
    assert np.array_equal(got[untouched], before[untouched])


def test_warm_up_is_bit_identical_to_no_buffer():
    T, Bf = 4, 4
    plain, buffered = Learner(_atari), Learner(_atari, replay=_prio_buffer(64, 4, seed=1, min_size=12))
    for k in range(3):
        batch, state = _batch(T, Bf, seed=10 + k), _state(2, Bf, 512 + A + 1, seed=k)
        assert not buffered.model.replay.mixing(Bf)
        sp, sb = plain.learn(batch, state), buffered.learn(batch, state)
        assert sp == sb
        assert torch.equal(plain.model.flat_params, buffered.model.flat_params)
    buf = buffered.model.replay
    assert buf.size == 12 and torch.all(buf.priorities[:12] > 0) and torch.all(buf.priorities[12:] == 0)


def _learn_step(run, batch, state, fresh=None, draw=None):
    from torchbeast_b200 import learner
    stats = learner.learn_step(run.flags, run.model, run.actor, batch, state, run.opt, None, fresh_columns=fresh,
                               draw=draw)
    torch.cuda.synchronize()
    return stats


CASES = {
    "atari_stacked": (_atari, dict(), (2, 512 + A + 1)),
    "atari_unstacked": (_atari, dict(frames="unstacked"), (2, 512 + A + 1)),
    "resnet_3x64x64": (_resnet, dict(obs=(3, 64, 64)), (1, 256)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_eager_learn_equals_learn_step_on_assembled_batch(case):
    from torchbeast_b200.replay import Draw
    make, kw, (layers, H) = CASES[case]
    T, Bf, R, cap = 4, 4, 6, 13
    run = Learner(make, replay=_prio_buffer(cap, R, seed=21, min_size=4))
    ref = Learner(make)
    shadow = Shadow(cap)
    buf = run.model.replay
    for k in range(4):                          # one warm-up step, three mixing steps
        batch, state = _batch(T, Bf, seed=40 + k, **kw), _state(layers, Bf, H, seed=k)
        mixing = buf.mixing(Bf)
        assert mixing == (k > 0)
        stats = run.learn(batch, state)
        leaves = {key: v for key, v in batch.items() if key in KEYS}
        leaves.update(h=state[0], c=state[1])
        want = shadow.call(leaves, Bf, R, mixing, buf.last_slots if mixing else None)
        if mixing:
            mb = {key: v for key, v in want.items() if key not in ("h", "c")}
            w = torch.cat([torch.ones(Bf, device="cuda"), buf.last_weights])
            assert torch.all(buf.last_weights > 0) and torch.all(buf.last_weights <= 1)
            ref_stats = _learn_step(ref, mb, (want["h"], want["c"]), fresh=Bf, draw=Draw(None, w, None))
        else:
            ref_stats = _learn_step(ref, batch, state)
        for key in LOSS_KEYS:
            assert stats[key] == ref_stats[key], (k, key)
        assert stats["episode_returns"] == ref_stats["episode_returns"]
        assert torch.equal(run.model.flat_params, ref.model.flat_params), k
        written = (buf.head - Bf + np.arange(Bf)) % cap
        assert torch.all(buf.priorities[torch.from_numpy(written).cuda()] > 0)


def _ring_copy(buf):
    return ([r.clone() for r in buf.rings], buf.state.clone(), (buf.head, buf.size, buf.seed, buf.step),
            buf.priorities.clone())


def _assert_same_buffer(a, b):
    assert a[2] == b[2]
    assert torch.equal(a[1], b[1])
    assert all(torch.equal(x, y) for x, y in zip(a[0], b[0]))
    assert torch.equal(a[3], b[3])


def test_graphed_equals_eager_and_follows_exponents_without_capture():
    T, Bf, R, cap = 4, 4, 6, 14
    runs = {g: Learner(_atari, graph=g, replay=_prio_buffer(cap, R, seed=8, min_size=8)) for g in (False, True)}
    for k in range(9):                          # warm-up for 2 steps, then mixing; the ring is full from step 4
        batch, state = _batch(T, Bf, seed=60 + k), _state(2, Bf, 512 + A + 1, seed=k)
        if k == 5:
            for r in runs.values():
                r.model.replay.importance_exponent = 1.0
        if k == 7:
            for r in runs.values():
                r.model.replay.priority_exponent = 0.0
        mixing = runs[True].model.replay.mixing(Bf)
        assert mixing == (k >= 2)
        se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
        for key in LOSS_KEYS:
            assert se[key] == sg[key], (k, key)
        assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params), k
        _assert_same_buffer(_ring_copy(runs[False].model.replay), _ring_copy(runs[True].model.replay))
        if mixing:
            e, g = runs[False].model.replay, runs[True].model.replay
            assert torch.equal(e.last_slots, g.last_slots) and torch.equal(e.last_weights, g.last_weights)
            if k >= 7:                          # alpha = 0: uniform draws, unit weights
                assert torch.all(g.last_weights == 1.0)
    assert len(runs[True].model._tb_graphs) == 2     # one graph per phase


@pytest.mark.parametrize("fill_calls", [1, 3])
def test_capture_leaves_the_buffer_untouched(fill_calls):
    from torchbeast_b200 import learner
    T, Bf, R, cap = 4, 4, 4, 10
    run = Learner(_atari, graph=True, replay=_prio_buffer(cap, R, seed=2, min_size=4))
    buf = run.model.replay
    for k in range(fill_calls):                 # plain learn calls: the priorities get values
        run.flags.cuda_graph = False
        run.learn(_batch(T, Bf, seed=80 + k), _state(2, Bf, 512 + A + 1, seed=k))
    run.flags.cuda_graph = True
    assert buf.size == min(fill_calls * Bf, cap)
    before = _ring_copy(buf)
    params = run.model.flat_params.clone()
    learner.GraphedLearner(run.flags, run.model, run.actor, run.opt, _batch(T, Bf, seed=90),
                           _state(2, Bf, 512 + A + 1, seed=9))
    torch.cuda.synchronize()
    _assert_same_buffer(before, _ring_copy(buf))
    assert torch.equal(params, run.model.flat_params)


def test_host_batch_and_polybeast_queue_match_device_path():
    from torchbeast_b200 import polybeast_learner
    T, Bf = 4, 4
    mk = lambda: _prio_buffer(10, 4, seed=6, min_size=4)   # noqa: E731
    dev_run, host_run, poly_run = Learner(_atari, replay=mk()), Learner(_atari, replay=mk()), Learner(_atari, replay=mk())
    batches = []
    for k in range(3):
        b = _batch(T, Bf, seed=70 + k)
        del b["last_action"]
        batches.append((b, _state(2, Bf, 512 + A + 1, seed=k)))
    for b, s in batches:
        dev_run.learn(b, s)
        host_run.learn({k: v.cpu() for k, v in b.items()}, tuple(x.cpu() for x in s))
    assert torch.equal(dev_run.model.flat_params, host_run.model.flat_params)
    _assert_same_buffer(_ring_copy(dev_run.model.replay), _ring_copy(host_run.model.replay))

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


@pytest.mark.parametrize("graph", [False, True])
def test_popart_with_prioritized_buffer_raises(graph):
    from torchbeast_b200 import polybeast_learner
    from torchbeast_b200._lib import TorchBeastB200Error

    def make():
        m = polybeast_learner.Net(A, True, observation_shape=(3, 64, 64), num_tasks=2)
        m.reset_parameters_like_torch(seed=3)
        return m
    run = Learner(make, graph=graph, replay=_prio_buffer(12, 4, seed=1, min_size=4))
    with pytest.raises(TorchBeastB200Error, match="PopArt"):
        run.learn(_batch(4, 4, seed=1, obs=(3, 64, 64), num_tasks=2), _state(1, 4, 256, seed=1))
    assert run.model.replay.size == 0
