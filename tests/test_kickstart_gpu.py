"""GPU: the kickstarting launch (tb_kickstart_loss_f32) against the float64 oracle of tests/kickstart_oracle.py over
T, B and A (the dynamic-A path included), weighted and unweighted, with -inf teacher logits; its bit properties (a zero
cost, identical logits, run to run); learn() with a teacher against a float64 autograd restatement for three
learner / teacher pairs; a teacher that is a copy of the learner; eager against graphed with the cost and the teacher's
weights changed between replays, over replay, the trust region, UPGO and two alternating batch shapes; and
polybeast_learner.learn through a LearnerQueue."""
import math
import types

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests import kickstart_oracle as KO
from tests.test_replay_gpu import FLAGS, LOSS_KEYS, _batch, _collect_graphs, _state  # noqa: F401

pytestmark = pytest.mark.gpu

A = 6
# (T, B, A): T in {1, 80, 600}, B in {1, 33, 8192} (8192 columns: a multi-CTA grid sum), A in {3, 6, 18}, and 11 and
# 23 on the dynamic-A path
SHAPES = [(1, 1, 3), (1, 33, 18), (1, 8192, 6), (80, 1, 6), (80, 33, 3), (80, 8192, 18), (600, 1, 18), (600, 33, 6),
          (600, 8192, 3), (80, 33, 11), (1, 8192, 23), (600, 33, 23)]


def _logits(T, B, A_, seed, masked=False):
    rs = np.random.RandomState(seed)
    teacher, target = (2 * rs.randn(T, B, A_)).astype(np.float32), (2 * rs.randn(T, B, A_)).astype(np.float32)
    if masked:
        teacher[:, ::3, 0] = -np.inf            # an illegal action in every third column
        teacher[0, 0, 1:] = -np.inf             # a one-hot teacher row
        teacher[0, 0, 0] = 0.0
    return teacher, target


def _run(teacher, target, cost, weights=None, grad_rows=1, seed=0):
    """One kickstart_loss on host inputs, into a pre-filled random grad_logits [T+grad_rows, B, A] and losses [4].
    Returns host copies of (before, after) for grad_logits and losses, and the Kickstart pair."""
    from torchbeast_b200 import learner
    T, B, A_ = target.shape
    rs = np.random.RandomState(seed + 1)
    gl = torch.from_numpy(rs.randn(T + grad_rows, B, A_).astype(np.float32)).cuda()
    losses = torch.from_numpy(rs.randn(4).astype(np.float32)).cuda()
    gl0, l0 = gl.clone(), losses.clone()
    cw = None if weights is None else torch.from_numpy(weights).cuda()
    ks = learner.kickstart_loss(torch.from_numpy(teacher).cuda(), torch.from_numpy(target).cuda(), losses, gl, cost,
                                column_weights=cw)
    torch.cuda.synchronize()
    h = lambda t: t.cpu().numpy()   # noqa: E731
    return dict(gl0=h(gl0), gl=h(gl), l0=h(l0), losses=h(losses), loss=h(ks.loss)[0], kl_sum=h(ks.kl_sum)[0])


def _check(out, o, cost, T):
    N = o["kl"].size
    kl_scale = np.abs(o["kl"]).sum()
    assert abs(float(out["kl_sum"]) - o["kl_sum"]) <= 2e-5 * kl_scale + 2e-6 * N
    assert abs(float(out["loss"]) - o["loss"]) <= cost * (2e-5 * kl_scale + 2e-6 * N)
    # exactly the term is added into rows t < T; row T is untouched
    added = out["gl"][:T].astype(np.float64) - out["gl0"][:T].astype(np.float64)
    np.testing.assert_allclose(added, o["grad_logits"], rtol=1e-4, atol=4e-6)
    assert np.array_equal(out["gl"][T:].view(np.int32), out["gl0"][T:].view(np.int32))
    # losses[3] gains the loss as float(double(total) + double(loss)); losses[:3] are untouched
    want = np.float32(np.float64(out["l0"][3]) + np.float64(out["loss"]))
    assert out["losses"][3].view(np.int32) == want.view(np.int32)
    assert np.array_equal(out["losses"][:3].view(np.int32), out["l0"][:3].view(np.int32))


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("T,B,A_", SHAPES)
def test_kernel_matches_float64_oracle(T, B, A_, weighted):
    seed = 7 * T + B + A_ + weighted
    teacher, target = _logits(T, B, A_, seed, masked=A_ in (6, 23))
    w = np.random.RandomState(seed).rand(B).astype(np.float32) if weighted else None
    if weighted and B > 2:
        w[1] = 0.0
    cost = 0.7
    out = _run(teacher, target, cost, weights=w, seed=seed)
    o = KO.loss(teacher, target, cost, weights=w)
    assert np.all(np.isfinite(o["kl"]))
    _check(out, o, cost, T)


def test_minus_inf_teacher_rows_give_no_nan():
    T, B, A_ = 20, 40, 6
    teacher, target = _logits(T, B, A_, 3)
    teacher[:, :, 2:5] = -np.inf
    teacher[5, 7, :] = -np.inf
    teacher[5, 7, 0] = 1.0                       # a one-hot teacher row
    out = _run(teacher, target, 1.5)
    o = KO.loss(teacher, target, 1.5)
    assert np.isfinite(out["kl_sum"]) and np.isfinite(out["loss"]) and np.all(np.isfinite(out["gl"]))
    _check(out, o, 1.5, T)


def test_grad_of_T_rows_and_forward_only():
    from torchbeast_b200 import learner
    T, B, A_ = 9, 5, 6
    teacher, target = _logits(T, B, A_, 4)
    full = _run(teacher, target, 0.5, grad_rows=1)
    exact = _run(teacher, target, 0.5, grad_rows=0)
    assert np.array_equal((full["gl"][:T] - full["gl0"][:T]).view(np.int32),
                          (exact["gl"] - exact["gl0"]).view(np.int32))
    losses = torch.zeros(4, device="cuda")
    ks = learner.kickstart_loss(torch.from_numpy(teacher).cuda(), torch.from_numpy(target).cuda(), losses, None, 0.5)
    assert ks.loss.item() == full["loss"] and ks.kl_sum.item() == full["kl_sum"]


def test_bit_properties():
    T, B, A_ = 80, 300, 6
    teacher, target = _logits(T, B, A_, 11)
    w = np.random.RandomState(2).rand(B).astype(np.float32)
    # a zero cost writes neither grad_logits nor losses; the KL sum is still reported
    z = _run(teacher, target, 0.0, weights=w)
    assert np.array_equal(z["gl"].view(np.int32), z["gl0"].view(np.int32))
    assert np.array_equal(z["losses"].view(np.int32), z["l0"].view(np.int32))
    assert z["loss"] == 0.0 and z["kl_sum"] > 0
    # identical logits: KL 0 and a gradient of +-0 exactly
    same = _run(target, target, 1.0, weights=w)
    assert same["loss"] == 0.0 and same["kl_sum"] == 0.0
    assert np.array_equal(same["gl"], same["gl0"]) and same["losses"][3] == same["l0"][3]
    # two runs are bit-identical, and the device-scalar cost gives the float's bits
    a, b = _run(teacher, target, 0.5, weights=w), _run(teacher, target, 0.5, weights=w)
    c = _run(teacher, target, torch.tensor([0.5], device="cuda"), weights=w)
    for k in ("gl", "losses", "loss", "kl_sum"):
        assert np.array_equal(np.asarray(a[k]).view(np.int32), np.asarray(b[k]).view(np.int32)), k
        assert np.array_equal(np.asarray(a[k]).view(np.int32), np.asarray(c[k]).view(np.int32)), k


# ---- learn() with a teacher ---------------------------------------------------------------------------------------


def _net(kind, use_lstm, seed, precision="fp32"):
    from torchbeast_b200 import monobeast, polybeast_learner
    if kind == "atari":
        m = monobeast.AtariNet((4, 84, 84), A, use_lstm, precision=precision)
    else:
        m = polybeast_learner.Net(A, use_lstm, precision=precision)
    m.reset_parameters_like_torch(seed=seed)
    return m


def _oracle_forward(kind, params, b, state):
    """(logits, baseline) of the float64 oracle net on host batch `b`."""
    if kind == "atari":
        return LT.atarinet_forward(params, b["frame"], b["reward"], b["done"], b["last_action"], state, A)[:2]
    return LT.resnet_forward(params, b["frame"], b["reward"], b["done"], state, A)[:2]


CASES = {
    "atari_lstm+atari_ff": (("atari", True), ("atari", False)),
    "resnet_lstm+resnet_lstm": (("resnet", True), ("resnet", True)),
    "resnet+atari_ff": (("resnet", False), ("atari", False)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_learn_matches_float64_autograd(case):
    from torchbeast_b200 import learner, optim
    from torchbeast_b200.kickstart import Teacher
    (lk, l_lstm), (tk, t_lstm) = CASES[case]
    T, B, cost = 5, 3, 0.8
    model, actor, tnet = _net(lk, l_lstm, 3), _net(lk, l_lstm, 3), _net(tk, t_lstm, 9)
    model.teacher = Teacher(tnet)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(**dict(FLAGS, grad_norm_clipping=1e9), kickstart_cost=cost)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=21, with_last_action=lk == "atari").items()}
    if lk == "atari":
        state = _state(2, B, 512 + A + 1, seed=4)
    else:
        state = _state(1, B, 256, seed=4) if l_lstm else ()
    p64 = {k: v.detach().double().cpu().requires_grad_(True) for k, v in model.state_dict().items()}
    t64 = {k: v.detach().double().cpu() for k, v in tnet.state_dict().items()}
    stats = learner.learn(flags, model, actor, batch, state, opt, None)
    torch.cuda.synchronize()
    # the float64 restatement: the learner's loss plus cost * sum KL(teacher || learner), by autograd
    hb = {k: v.cpu() for k, v in batch.items()}
    if "last_action" not in hb:
        hb["last_action"] = hb["action"]     # what learn() fills for the AtariNet teacher
    logits, baseline = _oracle_forward(lk, p64, hb, tuple(s.double().cpu() for s in state))
    with torch.no_grad():   # the teacher starts from its zero state
        t_state = tuple(torch.zeros(s.shape, dtype=torch.float64) for s in Teacher(tnet).initial_state(B))
        tlog, _ = _oracle_forward(tk, t64, hb, t_state)
    tl, vals = logits[:-1], baseline[:-1]
    rewards = hb["reward"][1:].double().clamp(-1, 1)
    discounts = (~hb["done"][1:]).double() * FLAGS["discounting"]
    vs, pg_adv, *_ = LT.vtrace_from_logits_torch(hb["policy_logits"][1:].double(), tl, hb["action"][1:], discounts,
                                                 rewards, vals, baseline[-1])
    pg, bl, en = LT.impala_losses_torch(tl, hb["action"][1:], pg_adv, vs, vals, FLAGS["baseline_cost"],
                                        FLAGS["entropy_cost"])
    lt, ls = torch.log_softmax(tlog[:-1], -1), torch.log_softmax(tl, -1)
    kl = (lt.exp() * (lt - ls)).sum(-1)
    ks = cost * kl.sum()
    total = pg + bl + en + ks
    names = list(p64)
    grads = torch.autograd.grad(total, [p64[n] for n in names], allow_unused=True)
    np.testing.assert_allclose(stats["total_loss"], total.item(), rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(stats["kickstart_loss"], ks.item(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(stats["teacher_kl"], kl.sum().item() / (T * B), rtol=1e-4, atol=1e-6)
    for n, g in zip(names, grads):
        ref = np.zeros(p64[n].shape) if g is None else g.numpy()
        got = dict(model.named_parameters())[n].grad.cpu().numpy()
        tol = 1e-4 * max(np.abs(ref).max(), 1e-6)
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=tol, err_msg=n)


@pytest.mark.parametrize("use_lstm", [False, True])
def test_a_copy_of_the_learner_as_teacher_changes_nothing(use_lstm):
    from torchbeast_b200 import learner, optim
    from torchbeast_b200.kickstart import Teacher
    runs = []
    for with_teacher in (False, True):
        model, actor = _net("atari", use_lstm, 3, "bf16x3"), _net("atari", use_lstm, 3, "bf16x3")
        opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
        flags = types.SimpleNamespace(**FLAGS)
        if with_teacher:
            twin = _net("atari", use_lstm, 77, "bf16x3")
            twin.load_state_dict({k: v.clone() for k, v in model.state_dict().items()})
            model.teacher = Teacher(twin)
            flags.kickstart_cost = 1.0
        stats = []
        for k in range(3):
            if with_teacher:   # the teacher follows the learner: a copy of its current weights
                twin.load_state_dict({n: v.clone() for n, v in model.state_dict().items()})
            batch = _batch(4, 4, seed=30 + k)
            stats.append(learner.learn(flags, model, actor, batch, model.initial_state(4), opt, None))
        torch.cuda.synchronize()
        runs.append((stats, model.flat_params.clone(), opt.snapshot()[0]))
    (s0, p0, o0), (s1, p1, o1) = runs
    assert torch.equal(p0, p1)
    assert len(o0) == len(o1) and all(torch.equal(a, b) for a, b in zip(o0, o1))
    for a, b in zip(s0, s1):
        for key in LOSS_KEYS:
            assert a[key] == b[key], key
        assert b["kickstart_loss"] == 0.0 and b["teacher_kl"] == 0.0


# ---- eager against graphed ------------------------------------------------------------------------------------------


class Run:
    """A learner with its own teacher; learn() eager or graphed."""

    def __init__(self, make, make_teacher, graph, replay=None, flags=None):
        from torchbeast_b200 import optim
        from torchbeast_b200.kickstart import Teacher
        self.model, self.actor = make(), make()
        self.model.teacher = Teacher(make_teacher())
        self.opt = optim.RMSprop(self.model, lr=0.00048, eps=0.01, alpha=0.99)
        self.flags = types.SimpleNamespace(cuda_graph=graph, **FLAGS, **(flags or {}))
        if replay is not None:
            self.model.replay = replay()

    def learn(self, batch, state):
        from torchbeast_b200 import learner
        stats = learner.learn(self.flags, self.model, self.actor, batch, state, self.opt, None)
        torch.cuda.synchronize()
        return stats


STATS = LOSS_KEYS + ("kickstart_loss", "teacher_kl")


def _compare(runs, batch, state, k, extra=()):
    se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
    assert set(se) == set(sg)
    for key in STATS + tuple(extra):
        assert se[key] == sg[key], (k, key)
    assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params), k
    return se


def _reload(runs, seed, make_teacher):
    """Load new teacher weights in place (one device copy into the flat buffer) into both runs' teachers."""
    src = make_teacher(seed)
    for r in runs.values():
        r.model.teacher.net.load_state_dict(src.state_dict())


NETS = {
    "atari": (lambda: _net("atari", True, 3, None), lambda seed=9: _net("atari", False, seed, None),
              lambda T, B, k, fr: (_batch(T, B, seed=40 + k, frames=fr), _state(2, B, 512 + A + 1, seed=k))),
    "resnet": (lambda: _net("resnet", True, 3, None), lambda seed=9: _net("atari", True, seed, None),
               lambda T, B, k, fr: (_batch(T, B, seed=40 + k, frames=fr), _state(1, B, 256, seed=k))),
}


@pytest.mark.parametrize("frames", ["stacked", "unstacked"])
@pytest.mark.parametrize("net", sorted(NETS))
def test_graphed_equals_eager_with_cost_and_teacher_weights_changed(net, frames):
    make, make_teacher, data = NETS[net]
    runs = {g: Run(make, make_teacher, g) for g in (False, True)}
    costs = [1.0, 1.0, 0.3, 0.0, 2.5, 0.7]
    for k, cost in enumerate(costs):
        for r in runs.values():
            r.flags.kickstart_cost = cost
        if k in (2, 4):
            _reload(runs, 100 + k, make_teacher)
        batch, state = data(4, 4, k, frames)
        se = _compare(runs, batch, state, k)
        if cost == 0.0:
            assert se["kickstart_loss"] == 0.0 and se["teacher_kl"] > 0
    assert len(runs[True].model._tb_graphs) == 1   # cost and weight changes captured nothing new
    # off: another graph, the stats lose the keys, and the step is the no-teacher step
    for r in runs.values():
        r.flags.kickstart_cost = None
    batch, state = data(4, 4, 99, frames)
    se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
    assert "kickstart_loss" not in se and "kickstart_loss" not in sg
    assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params)


def test_graphed_equals_eager_with_uniform_replay_warm_up_to_mixing():
    from torchbeast_b200.replay import ReplayBuffer
    make, make_teacher, data = NETS["atari"]
    runs = {g: Run(make, make_teacher, g, replay=lambda: ReplayBuffer(12, 4, seed=8, min_size=8),
                   flags=dict(kickstart_cost=0.9)) for g in (False, True)}
    for k in range(5):
        if k == 3:
            _reload(runs, 55, make_teacher)
        batch, state = data(4, 4, k, "stacked")
        _compare(runs, batch, state, k)
    assert len(runs[True].model._tb_graphs) == 2      # warm-up and mixing


def test_graphed_equals_eager_with_prioritised_replay_trust_region_and_upgo():
    from torchbeast_b200.replay import ReplayBuffer
    make, make_teacher, data = NETS["atari"]
    runs = {g: Run(make, make_teacher, g,
                   replay=lambda: ReplayBuffer(14, 4, seed=8, min_size=4, priority_exponent=0.6),
                   flags=dict(kickstart_cost=0.6, trust_region_kl=0.3, upgo_cost=0.8)) for g in (False, True)}
    for k in range(4):
        for r in runs.values():
            r.flags.kickstart_cost = (0.6, 0.0, 1.2, 0.4)[k]
        batch, state = data(4, 4, 70 + k, "stacked")
        _compare(runs, batch, state, k, extra=("upgo_loss", "trust_fraction", "mean_policy_kl"))
        assert torch.equal(runs[False].model.replay.priorities, runs[True].model.replay.priorities)


def test_two_batch_shapes_alternate_with_one_teacher():
    """Each graph replays into the teacher workspace it was captured with: the other shape's step replaces the
    teacher's buffers in between."""
    make, make_teacher, data = NETS["resnet"]
    runs = {g: Run(make, make_teacher, g, flags=dict(kickstart_cost=1.0)) for g in (False, True)}
    for k in range(6):
        B = (4, 6)[k % 2]
        batch, state = data(4, B, k, "stacked")
        _compare(runs, batch, state, k)
    assert len(runs[True].model._tb_graphs) == 2


def test_polybeast_learner_queue_matches_the_device_batch_path():
    from torchbeast_b200 import actors, learner, polybeast_learner
    T, B, steps = 4, 4, 3
    make, make_teacher, _ = NETS["atari"]
    nests, batches = [], []
    for k in range(steps):
        b = LT.synthetic_batch(T, B, A, seed=60 + k, with_last_action=False)
        state = tuple(s.cpu() for s in _state(2, B, 512 + A + 1, seed=k))
        env = (b["frame"], b["reward"], b["done"], torch.zeros(T + 1, B, dtype=torch.int32), b["episode_return"])
        nests.append(((env, (b["action"], b["policy_logits"], torch.zeros(T + 1, B))), state))
        batches.append(({k2: v.cuda() for k2, v in b.items()}, tuple(s.cuda() for s in state)))
    q = actors.LearnerQueue()
    for n in nests:
        q.put(n)
    q.close()
    poly, dev = Run(make, make_teacher, False, flags=dict(kickstart_cost=0.5)), \
        Run(make, make_teacher, False, flags=dict(kickstart_cost=0.5))
    poly.flags.unroll_length, poly.flags.batch_size = T, B
    log = []

    class Log:
        def log(self, s):
            log.append(dict(s))
    polybeast_learner.learn(poly.flags, q, poly.model, poly.actor, poly.opt, None, {}, Log())
    torch.cuda.synchronize()
    assert len(log) == steps
    for k, (batch, state) in enumerate(batches):
        s = learner.learn(dev.flags, dev.model, dev.actor, batch, state, dev.opt, None)
        for key in LOSS_KEYS + ("kickstart_loss", "teacher_kl"):
            assert log[k][key] == s[key], (k, key)
    torch.cuda.synchronize()
    assert torch.equal(poly.model.flat_params, dev.model.flat_params)


def test_without_a_cost_the_step_launches_what_it_did():
    from torchbeast_b200 import _lib
    make, make_teacher, data = NETS["atari"]
    counts, stats, params = {}, {}, {}
    for name, cost in (("absent", "absent"), ("none", None), ("on", 0.5)):
        run = Run(make, make_teacher, False)
        if name == "absent":
            run.model.teacher = None
        if cost not in ("absent", None):
            run.flags.kickstart_cost = cost
        batch, state = data(4, 4, 9, "stacked")
        run.learn(batch, state)                 # first step: one-time set-up launches
        before = _lib.lib().tb_launch_count()
        stats[name] = run.learn(batch, state)
        counts[name] = _lib.lib().tb_launch_count() - before
        params[name] = run.model.flat_params.clone()
    assert counts["none"] == counts["absent"] and counts["on"] > counts["absent"] + 1   # the teacher forward and the term
    assert "kickstart_loss" not in stats["none"] and "kickstart_loss" in stats["on"]
    assert torch.equal(params["none"], params["absent"])
    for key in LOSS_KEYS:
        assert stats["none"][key] == stats["absent"][key]


def test_invalid_cost_or_teacher_raises_before_any_launch():
    from torchbeast_b200 import _lib, monobeast
    from torchbeast_b200.kickstart import Teacher
    make, make_teacher, data = NETS["atari"]
    batch, state = data(4, 4, 1, "stacked")
    for graph in (False, True):
        for bad in ("nan", "actions", "self"):
            run = Run(make, make_teacher, graph, flags=dict(kickstart_cost=0.5))
            if bad == "nan":
                run.flags.kickstart_cost, err = math.nan, ValueError
            elif bad == "actions":
                run.model.teacher, err = Teacher(monobeast.AtariNet((4, 84, 84), A + 1)), _lib.TorchBeastB200Error
            else:
                run.model.teacher, err = Teacher(run.model), _lib.TorchBeastB200Error
            before = _lib.lib().tb_launch_count()
            params = run.model.flat_params.clone()
            with pytest.raises(err):
                run.learn(batch, state)
            assert _lib.lib().tb_launch_count() == before and torch.equal(params, run.model.flat_params), bad
