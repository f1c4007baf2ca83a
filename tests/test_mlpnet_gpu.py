"""GPU: MLPNet (vector observations).  The staging kernel bit for bit against its fp32 rule; forward and backward at
every precision against the float64 torch module of tests/mlpnet_oracle.py (flat, factored and Gaussian spaces, with
and without the LSTM, O = 3 .. 376, one to three hidden layers, normalisation on and off); the autograd forward against
learner_backward; one learn step against the existing loss oracles on the reference net's outputs (plain, PopArt, trust
region, UPGO, kickstarting with an MLPNet teacher, column weights); the running statistics against the NumPy merge;
eager against graphed learning with uniform and prioritised replay; and acting (seeded sampling, GraphedActor, the
polybeast inference loop)."""
import gc
import types

import numpy as np
import pytest
import torch

from tests import mlpnet_oracle as MO

pytestmark = pytest.mark.gpu

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


@pytest.fixture(autouse=True)
def _collect_graphs():
    yield
    gc.collect()
    torch.cuda.synchronize()


def _space(kind, A=6):
    from torchbeast_b200.action_space import Gaussian
    return {"flat": A, "factored": (3, 2, 4), "gaussian": Gaussian(3)}[kind]


def _oracle_space(kind):
    return {"flat": None, "factored": (3, 2, 4), "gaussian": ("gaussian", 3)}[kind]


def _net(O, kind, hidden, use_lstm, precision="fp32", norm=False, seed=0, tasks=None):
    from torchbeast_b200 import nets
    model = nets.MLPNet(O, _space(kind), hidden=hidden, use_lstm=use_lstm, precision=precision,
                        normalize_observations=norm, num_tasks=tasks)
    model.reset_parameters_like_torch(seed)
    if norm:  # statistics far from (0, 1), so the normalisation matters
        g = torch.Generator().manual_seed(seed + 1)
        model.obs_norm.mean.copy_(torch.randn(O, generator=g, dtype=torch.float64) * 3)
        model.obs_norm.var.copy_(torch.rand(O, generator=g, dtype=torch.float64) * 20 + 0.05)
        model.obs_norm.count.fill_(100.0)
    return model


def _batch(T1, B, O, kind, seed, model=None):
    """A rollout of T1 rows (T1 = T + 1 for a learn step); observations on features of very different scales."""
    g = torch.Generator().manual_seed(seed)
    scale = torch.logspace(-2, 2, O, dtype=torch.float64)
    frame = (torch.randn(T1, B, O, generator=g, dtype=torch.float64) * scale + 0.5).float()
    if model is not None and model.obs_norm is not None:
        n = model.obs_norm
        frame = (n.mean.cpu() + torch.randn(T1, B, O, generator=g, dtype=torch.float64) * n.var.cpu().sqrt() * 2).float()
        frame[0, 0, :] = n.mean.cpu().float() + 1e3  # clipped at +10
    if kind == "flat":
        act = torch.randint(0, 6, (T1, B), generator=g)
        logits = torch.randn(T1, B, 6, generator=g)
    elif kind == "factored":
        act = torch.stack([torch.randint(0, a, (T1, B), generator=g) for a in (3, 2, 4)], -1)
        logits = torch.randn(T1, B, 9, generator=g)
    else:
        logits = torch.cat([torch.randn(T1, B, 3, generator=g), torch.rand(T1, B, 3, generator=g) - 1.0], -1)
        act = logits[..., :3] + logits[..., 3:].exp() * torch.randn(T1, B, 3, generator=g)
    last = torch.cat([torch.zeros_like(act[:1]), act[:-1]], 0)
    b = dict(frame=frame, reward=torch.randn(T1, B, generator=g) * 2, done=torch.rand(T1, B, generator=g) < 0.1,
             episode_return=torch.randn(T1, B, generator=g), episode_step=torch.zeros(T1, B, dtype=torch.int32),
             policy_logits=logits, baseline=torch.randn(T1, B, generator=g), action=act, last_action=last)
    return {k: v.cuda() for k, v in b.items()}


def _state(model, B, seed=3):
    g = torch.Generator().manual_seed(seed)
    return tuple((0.3 * torch.randn(s.shape, generator=g)).cuda() for s in model.initial_state(B))


def _params64(model):
    return {name: p.detach().double().cpu().clone().requires_grad_(True) for name, p in model.named_parameters()}


def _reference(model, kind, batch, state, params=None):
    p = _params64(model) if params is None else params
    n = model.obs_norm
    logits, baseline, _ = MO.forward(
        p, batch["frame"].cpu(), batch["reward"].cpu(), batch["last_action"].cpu(), batch["done"].cpu(),
        tuple(s.cpu().double() for s in state) if state else None, model.hidden, model.num_actions,
        _oracle_space(kind), None if n is None else n.mean.cpu(), None if n is None else n.var.cpu())
    return p, logits, baseline


# ---- staging ---------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("O", [1, 17, 67])
@pytest.mark.parametrize("norm", [False, True])
def test_staging_matches_its_fp32_rule(precision, O, norm):
    from torchbeast_b200 import _lib
    N = 301
    g = torch.Generator().manual_seed(O)
    x = torch.randn(N, O, generator=g) * 30
    x[0, 0], x[1, 0], x[2, 0], x[3, 0] = float("nan"), float("inf"), float("-inf"), 1e-40
    mean = torch.randn(O, generator=g, dtype=torch.float64) * 5
    var = torch.rand(O, generator=g, dtype=torch.float64) * 4
    var[0] = 0.0
    y = MO.stage_f32(x, mean, var) if norm else x
    ld = O if precision == 0 else (O + 7) // 8 * 8
    planes = 2 if precision == 2 else 1
    out = torch.full((planes * N * ld,), -7, dtype=torch.float32 if precision == 0 else torch.bfloat16, device="cuda")
    p = _lib.ptr
    xd, md, vd = x.cuda(), mean.cuda(), var.cuda()  # held until the kernel has read them
    _lib.check(_lib.lib().tb_obs_stage(p(xd), N, O, p(md) if norm else None, p(vd) if norm else None, precision,
                                       p(out), _lib.stream_ptr()),
               "tb_obs_stage")
    got = out.cpu()
    if precision == 0:
        assert torch.equal(got.view(N, O).isnan(), y.isnan())
        assert torch.equal(torch.nan_to_num(got.view(N, O)).view(torch.int32), torch.nan_to_num(y).view(torch.int32))
        return
    pad = torch.zeros(N, ld)
    pad[:, :O] = y
    hi = pad.to(torch.bfloat16)
    want = [hi] + ([(pad - hi.float()).to(torch.bfloat16)] if precision == 2 else [])
    for k, w in enumerate(want):
        g_k = got[k * N * ld:(k + 1) * N * ld].view(N, ld)
        assert torch.equal(g_k.isnan(), w.isnan()), k
        assert torch.equal(torch.nan_to_num(g_k).view(torch.int16), torch.nan_to_num(w).view(torch.int16)), k


# ---- forward and backward --------------------------------------------------------------------------------------------

NET_CASES = [  # O, (T1, B), hidden, use_lstm, kind, norm
    (17, (5, 3), (256, 256), False, "flat", False),
    (3, (5, 3), (64,), True, "gaussian", True),
    (67, (81, 32), (128, 64, 32), False, "factored", True),
    (376, (81, 32), (256, 256), True, "flat", True),
    (17, (81, 32), (256, 256), True, "gaussian", False),
    (376, (5, 3), (32, 16, 8), True, "factored", False),
    (3, (81, 32), (8,), False, "flat", False),
    (67, (5, 3), (64, 64), True, "flat", True),
]


def _close(got, want, precision, what, below_relu=False):
    """fp32: elementwise.  bf16x3: elementwise, except for a torso gradient (`below_relu`), checked in norm: a
    pre-activation within the split-bf16 rounding of zero can flip its ReLU mask, and at N = 2592 rows a few do; each
    flip moves the gradients of its layer and of every layer below by one row's whole contribution, about 1/sqrt(N) of
    the sum (the split-bf16 GEMMs alone are within 1e-5 of float64 at these shapes).  bf16: in norm, the single-plane
    error of 2^-9 per product growing by sqrt(K) per layer the gradient crosses, and flipping masks far more often."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = max(np.abs(want).max(), 1e-30)
    err = np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30)
    if precision == "bf16":
        assert err < (0.3 if below_relu else 5e-2), (what, err)
    elif precision == "bf16x3" and below_relu:
        assert err < 2e-2, (what, err)
    else:
        np.testing.assert_allclose(got, want, rtol=2e-3, atol=2e-4 * scale, err_msg=what)


@pytest.mark.parametrize("precision", ["fp32", "bf16", "bf16x3"])
@pytest.mark.parametrize("case", range(len(NET_CASES)))
def test_forward_and_backward_match_float64(precision, case):
    O, (T1, B), hidden, use_lstm, kind, norm = NET_CASES[case]
    model = _net(O, kind, hidden, use_lstm, precision, norm, seed=case)
    batch = _batch(T1, B, O, kind, 10 + case, model)
    state = _state(model, B)
    out = model.learner_forward(batch, state)
    g = torch.Generator().manual_seed(case)
    gl = torch.randn(out.policy_logits.shape, generator=g)
    gb = torch.randn(out.baseline.shape, generator=g)
    fg = model.learner_backward(gl.cuda(), gb.cuda())
    torch.cuda.synchronize()
    p, logits, baseline = _reference(model, kind, batch, state)
    baseline = baseline[..., 0]
    (logits * gl.double()).sum().add((baseline * gb.double()).sum()).backward()
    _close(out.policy_logits.cpu(), logits.detach(), precision, "logits")
    _close(out.baseline.cpu(), baseline.detach(), precision, "baseline")
    for name, off, n, shape in [(nm, o, k, s) for (nm, _), (_, o, k, s) in zip(model._spec, model._views)]:
        _close(fg[off:off + n].view(shape).cpu(), p[name].grad, precision, name, below_relu=name.startswith("torso."))


def test_autograd_forward_equals_learner_backward():
    model = _net(17, "flat", (64, 32), True, "bf16x3", True, seed=4)
    batch = _batch(6, 5, 17, "flat", 5, model)
    state = _state(model, 5)
    out = model.learner_forward(batch, state)
    gl, gb = torch.randn_like(out.policy_logits), torch.randn_like(out.baseline)
    want = model.learner_backward(gl, gb).clone()
    model.zero_grad(set_to_none=True)
    o, _ = model(dict(batch), state)
    ((o["policy_logits"] * gl).sum() + (o["baseline"] * gb).sum()).backward()
    got = torch.cat([p.grad.reshape(-1) for p in model.parameters()])
    assert torch.equal(got, want)


# ---- one learn step against the loss oracles -------------------------------------------------------------------------


def _opt(model):
    from torchbeast_b200 import optim
    return optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)


@pytest.mark.parametrize("path", ["plain", "popart", "trust", "upgo", "kickstart", "weights"])
def test_learn_step_matches_the_loss_oracles(path):
    from oracle import vtrace_np as VO
    from oracle import learner_torch as LT
    from tests import kickstart_oracle as KO, popart_oracle as PO, trust_region_oracle as TR, upgo_oracle as UO
    from torchbeast_b200 import learner
    from torchbeast_b200.kickstart import Teacher
    T, B, O = 6, 4, 17
    model = _net(O, "flat", (64, 64), True, "fp32", True, seed=7, tasks=2 if path == "popart" else None)
    batch = _batch(T + 1, B, O, "flat", 8, model)
    state = _state(model, B)
    f = dict(FLAGS)
    teacher = None
    if path == "kickstart":
        teacher = _net(O, "flat", (32,), False, "fp32", True, seed=9)
        model.teacher = Teacher(teacher)
        f["kickstart_cost"] = 0.3
    if path == "upgo":
        f["upgo_cost"] = 0.7
    if path == "popart":
        batch["task"] = torch.randint(0, 2, (T + 1, B)).cuda()
    _, ref_logits, ref_base = _reference(model, "flat", batch, state)
    tl, n = ref_logits.detach().numpy(), ref_base.detach().numpy()
    bn = {k: v.cpu().numpy() for k, v in batch.items()}
    bl, acts, rw, dn = bn["policy_logits"][1:].astype(np.float64), bn["action"][1:], bn["reward"][1:], bn["done"][1:]
    if path == "trust":
        f["trust_region_kl"] = float(np.median(TR.policy_kl(bl, tl[:-1])))
    draw = None
    w = None
    if path == "weights":
        w = np.random.RandomState(3).uniform(0.2, 1.5, B).astype(np.float32)
        draw = types.SimpleNamespace(weights=torch.from_numpy(w).cuda(), buffer=None)
    mu, nu = (model.popart.mu.cpu(), model.popart.nu.cpu()) if path == "popart" else (None, None)
    step = learner.learn_step(types.SimpleNamespace(**f), model, None, batch, state, _opt(model), None,
                              stats_sync=False, draw=draw)
    torch.cuda.synchronize()
    losses, grad = step["losses"].cpu().numpy(), step["vtrace"].grad_logits.cpu().numpy()[:-1]
    tol = dict(rtol=1e-3, atol=1e-4)
    if path == "popart":
        t = torch.tensor(tl[:-1], requires_grad=True)
        want = PO.popart_losses(torch.from_numpy(bl), t, torch.from_numpy(acts), torch.from_numpy(rw),
                                torch.from_numpy(dn), torch.from_numpy(n.astype(np.float64)), batch["task"].cpu(), mu, nu,
                                hyper=LT.Hyper)
        want["total_loss"].backward()
        np.testing.assert_allclose(losses, [want[k].item() for k in ("pg_loss", "baseline_loss", "entropy_loss",
                                                                      "total_loss")], **tol)
        np.testing.assert_allclose(grad, t.grad.numpy(), rtol=1e-3, atol=1e-5)
        return
    values, boot = n[:-1, :, 0], n[-1, :, 0]
    disc = (~dn).astype(np.float64) * 0.99
    mask = None
    if path == "trust":
        mask = step["trust"].kl.cpu().numpy() <= f["trust_region_kl"]
    want = TR.loss(bl, tl[:-1], acts, np.clip(rw, -1, 1), disc, values, boot, mask=mask, entropy_cost=0.0006, weights=w)
    wl, wg = want["losses"].copy(), want["grad_logits"].copy()
    if path == "plain":  # the reference monobeast loss as well
        vo = VO.impala_loss(bl, tl[:-1], acts, rw, dn, values, boot)
        np.testing.assert_allclose(losses[3], vo.total_loss, **tol)
        np.testing.assert_allclose(grad, vo.grad_logits, rtol=1e-3, atol=1e-5)
    if path == "upgo":
        u = UO.loss(tl[:-1], acts, np.clip(rw, -1, 1), disc, values, boot, want["log_rhos"], 0.7)
        wl[3] += u["loss"]
        wg += u["grad_logits"]
    if path == "kickstart":
        p_t = dict(teacher.named_parameters())
        p_t = {k: v.detach().double().cpu() for k, v in p_t.items()}
        t_logits, _, _ = MO.forward(p_t, batch["frame"].cpu(), batch["reward"].cpu(), batch["last_action"].cpu(),
                                    hidden=teacher.hidden, num_actions=6, mean=teacher.obs_norm.mean.cpu(),
                                    var=teacher.obs_norm.var.cpu())
        k = KO.loss(t_logits.numpy()[:-1], tl[:-1], 0.3)
        wl[3] += k["loss"]
        wg += k["grad_logits"]
    np.testing.assert_allclose(losses, wl, **tol)
    np.testing.assert_allclose(grad, wg, rtol=1e-3, atol=1e-5)


# ---- running statistics ----------------------------------------------------------------------------------------------


def test_statistics_sums_skip_non_finite_entries_and_are_bit_identical():
    model = _net(5, "flat", (8,), False, norm=True)
    x = torch.randn(7, 300, 5) * 4 + 2
    x[3, 10, 1], x[4, 20, 1], x[5, 30, 2] = float("nan"), float("inf"), float("-inf")
    x[0] = 1e9  # row 0 is not counted
    frame = x.cuda()
    a, b = model.obs_norm_sums(frame, 250), model.obs_norm_sums(frame, 250)
    assert torch.equal(a, b)
    rows = x[1:, :250].reshape(-1, 5).double().numpy()
    fin = np.isfinite(rows)
    z = np.where(fin, rows, 0)
    np.testing.assert_array_equal(a[0].cpu().numpy(), fin.sum(0))
    np.testing.assert_allclose(a[1].cpu().numpy(), z.sum(0), rtol=1e-12)
    np.testing.assert_allclose(a[2].cpu().numpy(), (z * z).sum(0), rtol=1e-12)


@pytest.mark.parametrize("replay", [None, "uniform"])
def test_statistics_follow_the_fresh_rows(replay):
    from torchbeast_b200 import learner
    from torchbeast_b200.replay import ReplayBuffer
    T, B, O, steps = 5, 4, 17, 5
    from torchbeast_b200 import nets
    model = nets.MLPNet(O, 6, hidden=(32,), use_lstm=True, precision="fp32", normalize_observations=True)
    actor = nets.MLPNet(O, 6, hidden=(32,), use_lstm=True, precision="fp32", normalize_observations=True)
    if replay:
        model.replay = ReplayBuffer(8, 2, seed=5, min_size=2, stream_id=0)
    count, mean, var = np.zeros(O), np.zeros(O), np.ones(O)
    opt = _opt(model)
    for s in range(steps):
        batch = _batch(T + 1, B, O, "flat", 40 + s)
        batch["frame"][0] = 1e6  # row 0 repeats the previous rollout's last frame: not counted
        learner.learn(types.SimpleNamespace(**FLAGS), model, actor, batch, model.initial_state(B), opt, None)
        count, mean, var = MO.merge(count, mean, var, batch["frame"][1:].reshape(-1, O).double().cpu().numpy())
    n = model.obs_norm
    np.testing.assert_array_equal(n.count.cpu().numpy(), count)
    np.testing.assert_allclose(n.mean.cpu().numpy(), mean, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(n.var.cpu().numpy(), var, rtol=1e-12)
    for a, b in zip(actor.obs_norm.tensors(), n.tensors()):
        assert torch.equal(a, b)
    assert torch.equal(actor.flat_params, model.flat_params)
    # the state_dict round trip gives the same forward, bit for bit
    other = _net(O, "flat", (32,), True, norm=True, seed=11)
    other.load_state_dict({k: v.cpu() for k, v in model.state_dict().items()})
    b = _batch(3, B, O, "flat", 99)
    st = model.initial_state(B)
    assert torch.equal(other.learner_forward(b, st).policy_logits, model.learner_forward(b, st).policy_logits)


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(
        np.where(np.isnan(a), 0, a).view(np.int64), np.where(np.isnan(b), 0, b).view(np.int64))


@pytest.mark.parametrize("kind", ["flat", "gaussian"])
@pytest.mark.parametrize("replay", [None, "uniform", "prioritised"])
def test_learning_eager_equals_graphed(kind, replay):
    from torchbeast_b200 import learner
    from torchbeast_b200.replay import ReplayBuffer
    T, B, O, steps = 8, 4, 17, 6
    batches = [_batch(T + 1, B, O, kind, 60 + s) for s in range(steps)]
    runs = []
    for graphed in (False, True):
        model = _net(O, kind, (64, 64), True, "bf16x3", True, seed=3)
        actor = _net(O, kind, (64, 64), True, "bf16x3", True, seed=3)
        if replay is not None:
            model.replay = ReplayBuffer(6, 2, seed=5, min_size=2, stream_id=0,
                                        priority_exponent=0.6 if replay == "prioritised" else None)
        opt = _opt(model)
        f = types.SimpleNamespace(**FLAGS, cuda_graph=graphed, trust_region_kl=2.0)
        state = model.initial_state(B)
        stats = [learner.learn(f, model, actor, b, state, opt, None) for b in batches]
        runs.append((stats, model.flat_params.cpu().numpy(), [t.cpu().numpy() for t in model.obs_norm.tensors()],
                     actor.flat_params.cpu().numpy(), [t.cpu().numpy() for t in actor.obs_norm.tensors()]))
    for s0, s1 in zip(runs[0][0], runs[1][0]):
        assert s0.keys() == s1.keys()
        for k in s0:
            assert _bits_equal(np.asarray(s0[k], np.float64), np.asarray(s1[k], np.float64)), k
    assert _bits_equal(runs[0][1], runs[1][1]) and _bits_equal(runs[0][3], runs[1][3])
    for a, b in zip(runs[0][2] + runs[0][4], runs[1][2] + runs[1][4]):
        assert _bits_equal(a, b)
    assert np.all(np.isfinite([s["total_loss"] for s in runs[0][0]]))
    assert runs[0][2][2][0] == 100 + steps * T * B  # every fresh row counted once, no replayed one


# ---- acting ----------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["flat", "factored", "gaussian"])
def test_seeded_sampling_matches_the_oracles(kind):
    from oracle import sampling_np as SO
    from tests import factored_oracle as FO, gaussian_oracle as GO
    from torchbeast_b200.sampling import ActionSampler
    model = _net(17, kind, (64,), True, "bf16x3", True, seed=5)
    model.train()
    batch = _batch(1, 64, 17, kind, 6, model)
    model.action_sampler = ActionSampler(21, 4)
    with torch.no_grad():
        out, _ = model({k: batch[k] for k in ("frame", "reward", "done", "last_action")}, _state(model, 64))
    x = out["policy_logits"].cpu().numpy()
    a = out["action"].cpu().numpy()
    if kind == "flat":
        want, margin = SO.sample_actions(x, 21, 4)
        ok = margin >= SO.margin_threshold(6)
        assert ok.mean() > 0.9 and np.array_equal(a[ok], want[ok])
    elif kind == "factored":
        want, margin = FO.sample_actions(x, (3, 2, 4), 21, 4)
        ok = margin >= SO.margin_threshold(4)
        assert ok.mean() > 0.9 and np.array_equal(a[ok], want[ok])
    else:
        want, z = GO.sample(x.astype(np.float64), 21, 4)
        assert np.all(np.abs(a - want) <= GO.sample_tolerance(x.astype(np.float64), z))
    model.eval()
    with torch.no_grad():
        g, _ = model({k: batch[k] for k in ("frame", "reward", "done", "last_action")}, _state(model, 64))
    if kind == "gaussian":
        assert torch.equal(g["action"], g["policy_logits"][..., :3])
    elif kind == "flat":
        assert torch.equal(g["action"], g["policy_logits"].argmax(-1))


@pytest.mark.parametrize("B", [1, 48, 512])
def test_graphed_actor_matches_the_eager_forward(B):
    from torchbeast_b200.acting import GraphedActor, bucket_size
    from torchbeast_b200.sampling import ActionSampler
    model = _net(17, "gaussian", (64, 64), True, "bf16x3", True, seed=8)
    model.train()
    b = _batch(1, B, 17, "gaussian", 9, model)
    inputs = {k: b[k] for k in ("frame", "reward", "done", "last_action")}
    state = _state(model, B)
    actor = GraphedActor(model)
    Bk = bucket_size(B)
    pad = (lambda t: torch.cat([t, torch.zeros_like(t[:, :1]).expand(-1, Bk - B, *t.shape[2:])], 1)) if Bk > B \
        else (lambda t: t)
    for call in range(2):
        model.action_sampler = ActionSampler(31, 10 * call)
        with torch.no_grad():
            g_out, g_state = actor(inputs, state)
        model.action_sampler = ActionSampler(31, 10 * call)
        with torch.no_grad():
            e_out, e_state = model({k: pad(v) for k, v in inputs.items()}, tuple(pad(s) for s in state))
        for k in ("policy_logits", "baseline", "action"):
            assert torch.equal(g_out[k], e_out[k][:, :B]), k
        assert all(torch.equal(x, y[:, :B]) for x, y in zip(g_state, e_state))


def test_polybeast_inference_takes_vector_frames():
    from torchbeast_b200 import polybeast_learner
    model = _net(17, "flat", (64,), True, "bf16x3", True, seed=1)
    model.eval()
    B = 5
    b = _batch(1, B, 17, "flat", 2, model)
    got = []

    class Batch:
        def get_inputs(self):
            env = (b["frame"].cpu(), b["reward"].cpu(), b["done"].cpu(), torch.zeros(1, B, dtype=torch.int32),
                   torch.zeros(1, B), b["last_action"].cpu())
            return env, tuple(s.cpu() for s in model.initial_state(B))

        def set_outputs(self, outputs):
            got.append(outputs)

    polybeast_learner.inference(types.SimpleNamespace(), [Batch()], model)
    (action, logits, baseline), _ = got[0]
    assert action.shape == (1, B) and logits.shape == (1, B, 6) and baseline.shape == (1, B)
    assert torch.equal(action, logits.argmax(-1))
