"""GPU: the graphed learner follows loss and optimizer hyper-parameter changes between replays.  Every replay is
bit-identical to the eager step with the same values, a value that only feeds a kernel reuses the graph, and a value
that chooses a kernel or a buffer captures another one.  Also: the *_hp entry points against the float-argument ones."""
import gc
import types

import pytest
import torch

from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)
A = 6
T, B, STEPS = 8, 4, 6
LOSS_KEYS = ("total_loss", "pg_loss", "baseline_loss", "entropy_loss")


@pytest.fixture(autouse=True)
def _collect_graphs():
    """Models and the GraphedLearners stored on them reference each other: collect them between tests, so that no
    collection runs inside a later test's stream capture."""
    yield
    gc.collect()
    torch.cuda.synchronize()


def _net(seed=3):
    from torchbeast_b200 import monobeast
    m = monobeast.AtariNet((4, 84, 84), A, True)
    m.reset_parameters_like_torch(seed=seed)
    return m


def _batches(n, seed, done_dtype=torch.bool):
    out = []
    for i in range(n):
        b = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=seed + i, done_prob=0.2).items()}
        b["done"] = b["done"].to(done_dtype)
        out.append(b)
    return out


OPTS = [
    ("rmsprop", lambda m, o: o.RMSprop(m, lr=0.00048, momentum=0, eps=0.01, alpha=0.99)),
    ("rmsprop_centered_momentum_wd", lambda m, o: o.RMSprop(m, lr=4.8e-4, eps=0.01, alpha=0.99, centered=True,
                                                            momentum=0.5, weight_decay=1e-4)),
    ("adam", lambda m, o: o.Adam(m, lr=3e-4, weight_decay=0.01)),
    ("adamw", lambda m, o: o.AdamW(m, lr=3e-4)),
]


class Learner:
    """One model + actor + fused optimizer + LambdaLR + flags, stepped through monobeast.learn."""

    def __init__(self, make_opt, graph, seed=3, lr_decay=True):
        from torchbeast_b200 import optim
        self.model, self.actor = _net(seed), _net(seed)
        self.opt = make_opt(self.model, optim)
        self.sched = torch.optim.lr_scheduler.LambdaLR(self.opt, lambda k: 1.0 - k / 100.0) if lr_decay else None
        self.flags = types.SimpleNamespace(unroll_length=T, batch_size=B, cuda_graph=graph, **FLAGS)
        self.state = tuple(torch.zeros(2, B, 512 + A + 1, device="cuda") for _ in range(2))

    def learn(self, batch):
        from torchbeast_b200 import monobeast
        stats = monobeast.learn(self.flags, self.actor, self.model, batch, self.state, self.opt, self.sched)
        torch.cuda.synchronize()
        return stats


def _vary(k, flags, opt):
    """Step k's values: every loss value learn() reads and every non-structural value of the optimizer changes."""
    flags.entropy_cost = 0.0006 * (1 + k)
    flags.baseline_cost = 0.5 - 0.05 * k
    flags.discounting = 0.99 - 0.013 * k
    flags.reward_clipping = ("abs_one", "none")[k % 2]
    flags.grad_norm_clipping = (40.0, 0.5, None, 5.0, 1e-3, 100.0)[k % 6]  # active at 0.5 / 5 / 1e-3
    g = opt.param_groups[0]
    if "betas" in g:
        g["betas"] = (0.9 - 0.03 * k, 0.999 - 0.002 * k)
        g["eps"] = 1e-8 * 10.0 ** k
        g["weight_decay"] = (0.01, 0.0, 0.02, 0.05, 0.0, 0.001)[k % 6]
    else:
        g["alpha"] = 0.99 - 0.01 * k
        g["eps"] = 0.01 / (1 + k)
        if g["momentum"] != 0:
            g["momentum"] = 0.5 + 0.07 * k
        if g["weight_decay"] != 0:
            g["weight_decay"] = 1e-4 * (1 + k)


def _assert_same(eager, graphed, se, sg, what):
    assert torch.equal(eager.model.flat_params, graphed.model.flat_params), what
    assert torch.equal(graphed.actor.flat_params, graphed.model.flat_params), what
    for a, b in zip(eager.opt.flat_state(), graphed.opt.flat_state(), strict=True):
        assert torch.equal(a, b), what
    for key in LOSS_KEYS:
        assert se[key] == sg[key], (what, key, se[key], sg[key])
    assert se["episode_returns"] == sg["episode_returns"], what


def _graph_count(learner):
    return len(learner.model.__dict__.get("_tb_graphs", {}))


@pytest.mark.parametrize("make_opt", [c[1] for c in OPTS], ids=[c[0] for c in OPTS])
def test_changing_hparams_replay_equals_eager(make_opt):
    batches = _batches(STEPS, seed=70)
    eager, graphed = Learner(make_opt, graph=False), Learner(make_opt, graph=True)
    for k, b in enumerate(batches):
        for lrn in (eager, graphed):
            _vary(k, lrn.flags, lrn.opt)
        se, sg = eager.learn(b), graphed.learn(b)
        _assert_same(eager, graphed, se, sg, k)
        assert _graph_count(graphed) == 1
    # the LambdaLR moved the lr too (through the device scalar)
    assert eager.opt.param_groups[0]["lr"] == graphed.opt.param_groups[0]["lr"] < graphed.opt.defaults["lr"]
    if hasattr(graphed.opt, "step_device"):
        assert int(graphed.opt.step_device) == STEPS


def test_uint8_done_changing_discount_replay_equals_eager():
    batches = _batches(STEPS, seed=80, done_dtype=torch.uint8)
    make = OPTS[0][1]
    eager, graphed = Learner(make, graph=False), Learner(make, graph=True)
    for k, b in enumerate(batches):
        assert b["done"].dtype == torch.uint8 and bool(b["done"][1:].any())
        for lrn in (eager, graphed):
            _vary(k, lrn.flags, lrn.opt)
        se, sg = eager.learn(b), graphed.learn(b)
        _assert_same(eager, graphed, se, sg, k)
        assert _graph_count(graphed) == 1


def test_structural_change_captures_another_graph():
    """RMSprop weight_decay 0 -> 1e-4 switches the eager step to the _ex kernel: the graphed learner captures a second
    graph; back to 0 replays the first one again."""
    batches = _batches(STEPS, seed=90)
    make = OPTS[0][1]
    eager, graphed = Learner(make, graph=False), Learner(make, graph=True)
    wds = (0.0, 0.0, 1e-4, 2e-4, 0.0, 0.0)
    seen = []
    for k, b in enumerate(batches):
        for lrn in (eager, graphed):
            lrn.opt.param_groups[0]["weight_decay"] = wds[k]
            lrn.flags.entropy_cost = 0.0006 * (1 + k)
        se, sg = eager.learn(b), graphed.learn(b)
        _assert_same(eager, graphed, se, sg, k)
        current = [g for key, g in graphed.model._tb_graphs.items() if len(key) == 3]
        assert len(current) == 1
        seen.append(current[0])
        assert _graph_count(graphed) == (1 if k < 2 else 2), k
    assert seen[0] is seen[1] is seen[4] is seen[5]
    assert seen[2] is seen[3] and seen[2] is not seen[0]


def test_momentum_set_without_buffer_raises_before_capture_or_replay():
    from torchbeast_b200 import _lib
    b = _batches(2, seed=95)
    eager, graphed = Learner(OPTS[0][1], graph=False), Learner(OPTS[0][1], graph=True)
    graphed.learn(b[0])
    before = graphed.model.flat_params.clone()
    for lrn in (eager, graphed):
        lrn.opt.param_groups[0]["momentum"] = 0.9
    with pytest.raises(_lib.TorchBeastB200Error) as e_err:
        eager.learn(b[1])
    with pytest.raises(_lib.TorchBeastB200Error) as g_err:
        graphed.learn(b[1])
    assert str(g_err.value) == str(e_err.value) and "momentum needs a buffer" in str(g_err.value)
    assert _graph_count(graphed) == 1
    torch.cuda.synchronize()
    assert torch.equal(graphed.model.flat_params, before)
    # and before the first capture
    fresh = Learner(OPTS[0][1], graph=True)
    fresh.opt.param_groups[0]["momentum"] = 0.9
    with pytest.raises(_lib.TorchBeastB200Error, match="momentum needs a buffer"):
        fresh.learn(b[1])
    assert _graph_count(fresh) == 0


@pytest.mark.parametrize("make_opt", [OPTS[0][1], OPTS[2][1]], ids=["rmsprop", "adam"])
def test_population_based_training_exploit(make_opt):
    """Two members with captured graphs.  B exploits A: A's weights and optimizer state_dict are copied into B, B's lr,
    eps and entropy_cost are perturbed, and B steps on.  Its replays equal an eager twin's, with no new capture."""
    member_a, member_b = Learner(make_opt, graph=True, seed=5, lr_decay=False), \
        Learner(make_opt, graph=True, seed=6, lr_decay=False)
    for b in _batches(2, seed=100):
        member_a.learn(b)
    for b in _batches(2, seed=110):
        member_b.learn(b)
    assert _graph_count(member_a) == _graph_count(member_b) == 1
    twin = Learner(make_opt, graph=False, seed=7, lr_decay=False)
    for lrn in (member_b, twin):
        lrn.model.load_state_dict(member_a.model.state_dict())
        lrn.opt.load_state_dict(member_a.opt.state_dict())
        g = lrn.opt.param_groups[0]
        g["lr"] *= 1.2
        g["eps"] *= 0.8
        lrn.flags.entropy_cost *= 1.2
    assert torch.equal(member_b.model.flat_params, member_a.model.flat_params)
    for k, b in enumerate(_batches(3, seed=120)):
        se, sg = twin.learn(b), member_b.learn(b)
        _assert_same(twin, member_b, se, sg, k)
        assert _graph_count(member_b) == 1
    assert not torch.equal(member_b.model.flat_params, member_a.model.flat_params)


def _block(rec):
    from torchbeast_b200 import learner
    blk = torch.zeros(learner.HPARAMS.itemsize, dtype=torch.uint8, device="cuda")
    learner.publish_hparams(rec, blk)
    return blk


@pytest.mark.parametrize("clips", [(1.0, 1.0), (0.5, None), (None, 2.0)])
@pytest.mark.parametrize("done_dtype", [torch.bool, torch.uint8])
def test_loss_reads_the_block_bit_identically(clips, done_dtype):
    """impala_loss_fwd_bwd with hparams_dev equals the call with the same values as arguments, every output bit for bit,
    including the V-trace clip thresholds learn() does not change.  A uint8 `done` discounts by (255 - done) * gamma,
    as the reference's bitwise `~done` does, so its sequences are kept short enough to stay finite."""
    from torchbeast_b200 import learner
    g = torch.Generator().manual_seed(5)
    Tl, Bl, Al = (20 if done_dtype == torch.bool else 4), 40, 9
    bl, tl = torch.randn(Tl, Bl, Al, generator=g).cuda(), torch.randn(Tl, Bl, Al, generator=g).cuda()
    ac = torch.randint(0, Al, (Tl, Bl), generator=g).cuda()
    rw = (3 * torch.randn(Tl, Bl, generator=g)).cuda()
    dn = (torch.rand(Tl, Bl, generator=g) < 0.1).cuda().to(done_dtype)
    va, bs = torch.randn(Tl, Bl, generator=g).cuda(), torch.randn(Bl, generator=g).cuda()
    for clip_mode in ("abs_one", "none"):
        flags = types.SimpleNamespace(discounting=0.97, baseline_cost=0.3, entropy_cost=0.01, reward_clipping=clip_mode,
                                      grad_norm_clipping=None)
        want = learner.impala_loss_fwd_bwd(bl, tl, ac, rw, dn, va, bs, discounting=0.97, baseline_cost=0.3,
                                           entropy_cost=0.01, reward_clipping=clip_mode, clip_rho_threshold=clips[0],
                                           clip_pg_rho_threshold=clips[1])
        blk = _block(learner.pack_hparams(flags, None, clip_rho_threshold=clips[0], clip_pg_rho_threshold=clips[1]))
        got = learner.impala_loss_fwd_bwd(bl, tl, ac, rw, dn, va, bs, hparams_dev=blk)
        for name, a, b in zip(want._fields, want, got, strict=True):
            assert bool(torch.isfinite(a).all()), (clip_mode, name)
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (clip_mode, name)


OPT_STEP_CASES = [
    ("rmsprop", dict(lr=4.8e-4, alpha=0.95, eps=0.01)),
    ("rmsprop", dict(lr=4.8e-4, alpha=0.95, eps=0.01, momentum=0.9)),
    ("rmsprop", dict(lr=4.8e-4, eps=1e-4, weight_decay=0.05)),
    ("rmsprop", dict(lr=4.8e-4, eps=1e-4, centered=True, momentum=0.5, weight_decay=1e-3)),
    ("adam", dict(lr=1e-3, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.05)),
    ("adamw", dict(lr=1e-3, betas=(0.85, 0.995), weight_decay=0.05)),
]


@pytest.mark.parametrize("name,kw", OPT_STEP_CASES, ids=["%s%d" % (c[0], i) for i, c in enumerate(OPT_STEP_CASES)])
def test_optimizer_step_reads_the_block_bit_identically(name, kw):
    """Five steps of optimizer.step(hparams_dev=block) against optimizer.step(max_grad_norm) on a twin, with the clip
    active on some steps; launches and profile records are the same."""
    from torchbeast_b200 import _lib, learner, optim
    cls = {"rmsprop": optim.RMSprop, "adam": optim.Adam, "adamw": optim.AdamW}[name]
    m_arg, m_blk = _net(), _net()
    o_arg, o_blk = cls(m_arg, **kw), cls(m_blk, **kw)
    gen = torch.Generator(device="cuda").manual_seed(3)
    lib = _lib.lib()
    for k, max_norm in enumerate((40.0, 1.0, None, 0.25, 1e4)):
        gr = torch.randn(m_arg.flat_params.numel(), device="cuda", generator=gen) * (1 + k)
        flags = types.SimpleNamespace(discounting=0.99, baseline_cost=0.5, entropy_cost=0.0, reward_clipping="none",
                                      grad_norm_clipping=max_norm)
        blk = _block(learner.pack_hparams(flags, o_blk))
        records = []
        for m, o, hp in ((m_arg, o_arg, None), (m_blk, o_blk, blk)):
            m.attach_grads().copy_(gr)
            torch.cuda.synchronize()
            before = lib.tb_launch_count()
            lib.tb_profile_enable(1)
            o.step(max_grad_norm=max_norm, hparams_dev=hp)
            records.append(([n for n, _ in _lib.profile_collect()], lib.tb_launch_count() - before))
            lib.tb_profile_enable(0)
        assert records[0] == records[1], records
        assert torch.equal(m_arg.flat_params, m_blk.flat_params), k
        assert torch.equal(m_arg.flat_grad, m_blk.flat_grad), k
        assert torch.equal(o_arg.grad_norm, o_blk.grad_norm), k
        for a, b in zip(o_arg.flat_state(), o_blk.flat_state(), strict=True):
            assert torch.equal(a, b), k
