"""GPU: continuous (diagonal-Gaussian) action spaces.  tb_impala_loss_gaussian_f32 against the float64 oracle of
tests/gaussian_oracle.py on every feature path, both launch layouts and D = 1, 6, 21; the Gaussian sampler against
the oracle's Philox / Box-Muller rule, host against device (seed, step), its moments and its NaN rows; AtariNet's
continuous entries against a float64 torch restatement of the net (core input, forward and backward) and ResNet's
against its own entries at num_actions = 2D; learn_step against a float64 torch reference of the loss, eager against
graphed learning and acting, replay of float action leaves; and the cases that raise."""
import gc
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import gaussian_oracle as GO

pytestmark = pytest.mark.gpu

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.01, grad_norm_clipping=40.0)


@pytest.fixture(autouse=True)
def _collect_graphs():
    yield
    gc.collect()
    torch.cuda.synchronize()


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(
        np.where(np.isnan(a), 0, a).view(np.int32), np.where(np.isnan(b), 0, b).view(np.int32))


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _inputs(T, B, D, seed, K=None):
    """Behaviour rows, target rows near them, and actions drawn from the behaviour policy."""
    rs = np.random.RandomState(seed)
    bl = np.concatenate([rs.randn(T, B, D), rs.uniform(-1.0, 0.5, (T, B, D))], -1)
    tl = bl + 0.15 * rs.randn(T, B, 2 * D) / np.sqrt(D)
    mu, l = GO.split(bl)
    d = dict(bl=bl.astype(np.float32), tl=tl.astype(np.float32),
             actions=(mu + np.exp(l) * rs.randn(T, B, D)).astype(np.float32),
             rewards=(2 * rs.randn(T, B)).astype(np.float32), done=rs.rand(T, B) < 0.1,
             values=rs.randn(T, B).astype(np.float32), bootstrap=rs.randn(B).astype(np.float32),
             weights=rs.rand(B).astype(np.float32))
    if K is not None:
        d["n"] = rs.randn(T + 1, B, K).astype(np.float32)
        d["task"] = rs.randint(0, K, size=(T + 1, B)).astype(np.int64)
        d["mu"] = 0.3 * rs.randn(K)
        d["nu"] = d["mu"] ** 2 + 0.5 + rs.rand(K)
    # the trust region's beta: the median KL, so that some rows exceed it and some do not
    d["beta"] = float(np.median(GO.kl(d["tl"], d["bl"])))
    return d


def _run(d, D, path):
    """One loss call through learner.impala_loss_fwd_bwd / impala_loss_popart with action_space=Gaussian(D)."""
    from torchbeast_b200 import learner
    from torchbeast_b200.action_space import Gaussian
    kw = dict(discounting=0.99, baseline_cost=0.5, entropy_cost=0.01)
    beta = d["beta"] if "trust" in path else None
    hp = None
    if "hp" in path:
        rec = learner.pack_hparams(types.SimpleNamespace(grad_norm_clipping=None, reward_clipping="abs_one", **kw))
        hp = torch.zeros(learner.HPARAMS.itemsize, dtype=torch.uint8, device="cuda")
        learner.publish_hparams(rec, hp)
    if "popart" in path:
        res = learner.impala_loss_popart(_cu(d["bl"]), _cu(d["tl"]), _cu(d["actions"]), _cu(d["rewards"]),
                                         _cu(d["done"]), _cu(d["n"]), _cu(d["task"]), _cu(d["mu"]), _cu(d["nu"]),
                                         hparams_dev=hp, trust_region=beta, action_space=Gaussian(D), **kw)
        loss, sums = res[0], res[1]
        trust = res[2] if beta is not None else None
    else:
        res = learner.impala_loss_fwd_bwd(
            _cu(d["bl"]), _cu(d["tl"]), _cu(d["actions"]), _cu(d["rewards"]), _cu(d["done"]), _cu(d["values"]),
            _cu(d["bootstrap"]), hparams_dev=hp, trust_region=beta, action_space=Gaussian(D),
            column_weights=_cu(d["weights"]) if "weighted" in path else None, **kw)
        loss, trust = (res if beta is not None else (res, None))
        sums = None
    torch.cuda.synchronize()
    out = {k: getattr(loss, k).cpu().numpy() for k in loss._fields}
    if trust is not None:
        out["kl"], out["trust_out"] = trust.kl.cpu().numpy(), trust.sums.cpu().numpy()
    if sums is not None:
        out["task_sums"] = sums.cpu().numpy()
    return out


def _oracle(d, path):
    kw = dict(entropy_cost=0.01, trust_beta=d["beta"] if "trust" in path else None,
              weights=d["weights"] if "weighted" in path else None)
    if "popart" in path:
        return GO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], d["n"], None,
                              popart=(d["task"], d["mu"], d["nu"]), **kw)
    return GO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], d["values"], d["bootstrap"], **kw)


PATHS = ["plain", "hp", "weighted", "trust", "weighted_trust", "popart", "popart_trust"]


@pytest.mark.parametrize("D", [1, 6, 21])
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("T,B", [(80, 32), (4, 2)])  # split-T layout; single-launch layout
def test_loss_matches_the_oracle(D, path, T, B):
    d = _inputs(T, B, D, 100 + T + D, K=3 if "popart" in path else None)
    got, want = _run(d, D, path), _oracle(d, path)
    # fp32 log-densities are sums of D terms of magnitude ~ 1 + z^2: a few ulp each
    tol = dict(rtol=2e-4, atol=2e-5 * D)
    for k in ("log_rhos", "target_action_log_probs", "behavior_action_log_probs"):
        wk = {"target_action_log_probs": "target_alp", "behavior_action_log_probs": "behavior_alp"}.get(k, k)
        np.testing.assert_allclose(got[k], want[wk], err_msg=k, **tol)
    for k in ("vs", "pg_advantages"):
        np.testing.assert_allclose(got[k], want["pg_adv" if k == "pg_advantages" else k], rtol=2e-4, atol=2e-4,
                                   err_msg=k)
    np.testing.assert_allclose(got["losses"], want["losses"], rtol=2e-4, atol=1e-3)
    np.testing.assert_allclose(got["grad_logits"][:-1], want["grad_logits"], rtol=1e-3, atol=1e-4)
    assert np.all(got["grad_logits"][-1] == 0)
    gv = got["grad_values"]
    np.testing.assert_allclose(gv if "popart" in path else gv[:-1], want["grad_values"], rtol=1e-3, atol=1e-5)
    if "trust" in path:
        np.testing.assert_allclose(got["kl"], want["kl"], rtol=1e-4, atol=1e-5 * D)
        assert 0 < got["trust_out"][0] < T * B
        # rows within rounding of beta may land on either side
        near = np.abs(want["kl"] - d["beta"]) <= 1e-4 * (1 + d["beta"])
        assert abs(got["trust_out"][0] - want["trusted"]) <= near.sum()
    if "popart" in path:
        np.testing.assert_allclose(got["task_sums"], want["task_sums"], rtol=1e-4, atol=1e-3)


def test_non_finite_entries_poison_their_row():
    D = 3
    d = _inputs(6, 4, D, 3)
    d["tl"][2, 1, D + 1] = np.inf
    d["actions"][4, 0, 2] = np.nan
    got = _run(d, D, "plain")
    for t, b in ((2, 1), (4, 0)):
        assert np.isnan(got["target_action_log_probs"][t, b]) and np.isnan(got["grad_logits"][t, b]).all()
    assert np.isnan(got["losses"][3])
    alp = got["target_action_log_probs"].copy()
    alp[2, 1] = alp[4, 0] = 0
    assert np.isfinite(alp).all()


# ---- sampling --------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("D", [1, 6, 21, 64])
def test_sampler_matches_the_oracle(D):
    """mu = 0, l = 0 gives a = z: a sample within the fp32 tolerance of the oracle's means every Philox word is the
    contract's (one wrong bit above bit 8 moves z by far more); then random (mu, l) rows."""
    from torchbeast_b200.sampling import ActionSampler
    T, B = 3, 257
    ids = np.arange(B, dtype=np.int64) * 5 - 300
    for rows in (np.zeros((T, B, 2 * D), np.float32),
                 np.concatenate([np.random.RandomState(D).randn(T, B, D),
                                 np.random.RandomState(D + 1).uniform(-2, 1, (T, B, D))], -1).astype(np.float32)):
        s = ActionSampler(2 ** 33 + 5, 17)
        got = s.sample(_cu(rows), _cu(ids), continuous_dim=D).cpu().numpy()
        assert s.step == 17 + T and got.shape == (T, B, D) and got.dtype == np.float32
        want, z = GO.sample(rows, 2 ** 33 + 5, 17, ids)
        err = np.abs(got - want)
        assert np.all(err <= GO.sample_tolerance(rows, z)), err.max()


def test_sampler_host_and_device_seed_step_give_identical_bits_eager_and_graphed():
    from torchbeast_b200.sampling import sample_gaussian
    D, B = 6, 300
    y = _cu(np.random.RandomState(2).randn(1, B, 2 * D).astype(np.float32))
    ids = torch.arange(B, dtype=torch.int64, device="cuda") * 7 - 100
    seed_step = torch.zeros(2, dtype=torch.int64, device="cuda")
    sample_gaussian(y, D, ids, seed_step=seed_step)  # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = sample_gaussian(y, D, ids, seed_step=seed_step)
    for step in (0, 1, 12345):
        seed_step.copy_(torch.tensor([2 ** 40 + 3, step]))
        g.replay()
        torch.cuda.synchronize()
        host = sample_gaussian(y, D, ids, seed=2 ** 40 + 3, step=step)
        dev = sample_gaussian(y, D, ids, seed_step=seed_step)
        assert _bits_equal(out.cpu(), host.cpu()) and _bits_equal(dev.cpu(), host.cpu())


def test_sampler_moments():
    """2^20 draws per component: the sample mean lies within 5 standard errors (sigma / 2^10) of mu and the sample
    standard deviation within 5 of its standard errors (sigma / sqrt(2 N)) of sigma."""
    from torchbeast_b200.sampling import ActionSampler
    D, N = 4, 2 ** 20
    mu = np.array([0.0, -3.0, 1.5, 100.0], np.float32)
    l = np.array([0.0, -2.0, 1.0, -5.0], np.float32)
    rows = np.broadcast_to(np.concatenate([mu, l]), (64, N // 64, 2 * D))
    a = ActionSampler(7, 0).sample(_cu(rows.astype(np.float32)), continuous_dim=D).double().reshape(N, D)
    sig = np.exp(l.astype(np.float64))
    m, s = a.mean(0).cpu().numpy(), a.std(0).cpu().numpy()
    assert np.all(np.abs(m - mu) <= 5 * sig / np.sqrt(N)), (m, mu)
    assert np.all(np.abs(s - sig) <= 5 * sig / np.sqrt(2 * N)), (s, sig)


def test_sampler_non_finite_rows_give_nan():
    from torchbeast_b200.sampling import ActionSampler
    D = 3
    rows = np.random.RandomState(4).randn(2, 5, 2 * D).astype(np.float32)
    rows[0, 1, 0] = np.nan
    rows[1, 2, D + 2] = np.inf
    rows[1, 4, 1] = -np.inf
    got = ActionSampler(1, 0).sample(_cu(rows), continuous_dim=D).cpu().numpy()
    bad = np.zeros(got.shape, bool)
    bad[0, 1, 0] = bad[1, 2, 2] = bad[1, 4, 1] = True
    assert np.isnan(got[bad]).all() and np.isfinite(got[~bad]).all()


# ---- nets ------------------------------------------------------------------------------------------------------------


def _net(kind, D, use_lstm, seed, precision=None):
    from torchbeast_b200 import nets
    from torchbeast_b200.action_space import Gaussian
    m = (nets.AtariNet((4, 84, 84), Gaussian(D), use_lstm, precision=precision) if kind == "atari"
         else nets.ResNet(Gaussian(D), use_lstm, precision=precision))
    m.reset_parameters_like_torch(seed=seed)
    return m


def _batch(kind, T, B, D, seed):
    """A small synthetic task: the reward is higher the closer action component 0 is to 0.5."""
    g = torch.Generator().manual_seed(seed)
    action = torch.randn(T + 1, B, D, generator=g)
    b = dict(frame=torch.randint(0, 255, (T + 1, B, 4, 84, 84), generator=g, dtype=torch.uint8),
             reward=1.0 - (action[..., 0] - 0.5).abs(), done=torch.rand(T + 1, B, generator=g) < 0.1,
             episode_return=torch.randn(T + 1, B, generator=g),
             policy_logits=torch.cat([0.3 * torch.randn(T + 1, B, D, generator=g),
                                      torch.full((T + 1, B, D), -0.2)], -1),
             action=action)
    if kind == "atari":
        b["last_action"] = torch.cat([torch.zeros(1, B, D), action[:-1]])
    return {k: v.cuda() for k, v in b.items()}


def _state(model, B):
    g = torch.Generator().manual_seed(B)
    return tuple((0.1 * torch.randn(s.shape, generator=g)).cuda() for s in model.initial_state(B))


def _torch_atarinet(model, batch, state):
    """AtariNet restated in float64 torch (monobeast.py AtariNet.forward with the continuous core input): returns
    (core input, logits, baseline) with autograd to the float64 parameter copies in `params`."""
    params = {k: v.detach().double().requires_grad_() for k, v in model.state_dict().items()}
    T1, B = batch["reward"].shape
    x = batch["frame"].reshape(T1 * B, 4, 84, 84).double() / 255.0
    x = F.relu(F.conv2d(x, params["conv1.weight"], params["conv1.bias"], stride=4))
    x = F.relu(F.conv2d(x, params["conv2.weight"], params["conv2.bias"], stride=2))
    x = F.relu(F.conv2d(x, params["conv3.weight"], params["conv3.bias"], stride=1))
    x = F.relu(F.linear(x.reshape(T1 * B, -1), params["fc.weight"], params["fc.bias"]))
    r = batch["reward"].double().clamp(-1, 1).reshape(T1 * B, 1)
    core_in = torch.cat([x, r, batch["last_action"].double().reshape(T1 * B, -1)], -1)
    core_out = core_in
    if model.use_lstm:
        h, c = (s.double() for s in state)
        notdone = (~batch["done"]).double()
        outs = []
        seq = core_in.reshape(T1, B, -1)
        for t in range(T1):
            h, c = h * notdone[t][None, :, None], c * notdone[t][None, :, None]
            inp, hs, cs = seq[t], [], []
            for layer in range(2):
                gates = (F.linear(inp, params["core.weight_ih_l%d" % layer], params["core.bias_ih_l%d" % layer])
                         + F.linear(h[layer], params["core.weight_hh_l%d" % layer], params["core.bias_hh_l%d" % layer]))
                i, f, gg, o = gates.chunk(4, -1)
                cl = torch.sigmoid(f) * c[layer] + torch.sigmoid(i) * torch.tanh(gg)
                hl = torch.sigmoid(o) * torch.tanh(cl)
                hs.append(hl)
                cs.append(cl)
                inp = hl
            h, c = torch.stack(hs), torch.stack(cs)
            outs.append(inp)
        core_out = torch.stack(outs).reshape(T1 * B, -1)
    logits = F.linear(core_out, params["policy.weight"], params["policy.bias"]).reshape(T1, B, -1)
    baseline = F.linear(core_out, params["baseline.weight"], params["baseline.bias"]).reshape(T1, B)
    return params, core_in, logits, baseline


@pytest.mark.parametrize("use_lstm", [False, True])
def test_atarinet_continuous_forward_and_backward_match_a_torch_restatement(use_lstm):
    """precision fp32 (SIMT GEMMs): the core input (as the gradient of the policy logits reaching it, and through the
    logits), the logits, the baseline and every parameter gradient of tb_atarinet_backward_continuous against float64
    autograd of the same net."""
    T, B, D = 3, 4, 6
    model = _net("atari", D, use_lstm, 11, precision="fp32")
    batch = _batch("atari", T - 1, B, D, 12)
    batch["last_action"] = 3 * batch["last_action"]  # values a one-hot could not hold
    state = _state(model, B)
    out, _ = model(dict(batch), state)
    params, core_in, logits, baseline = _torch_atarinet(model, batch, state)
    assert core_in.shape[-1] == 512 + D + 1
    np.testing.assert_allclose(out["policy_logits"].detach().cpu().numpy(), logits.detach().cpu().numpy(),
                               rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(out["baseline"].detach().cpu().numpy(), baseline.detach().cpu().numpy(),
                               rtol=1e-4, atol=1e-4)
    g = torch.Generator().manual_seed(3)
    gl, gb = torch.randn(logits.shape, generator=g).cuda(), torch.randn(baseline.shape, generator=g).cuda()
    model.zero_grad(set_to_none=True)
    ((out["policy_logits"] * gl).sum() + (out["baseline"] * gb).sum()).backward()
    ((logits * gl.double()).sum() + (baseline * gb.double()).sum()).backward()
    for name, p in model.named_parameters():
        want = params[name].grad.cpu().numpy()
        scale = np.abs(want).max() + 1e-30
        np.testing.assert_allclose(p.grad.cpu().numpy(), want, rtol=1e-3, atol=1e-4 * scale, err_msg=name)
    # last_action enters the core as it is: its columns move the logits by policy.weight's columns (no LSTM), or at
    # least move them (LSTM).  After the backward: a forward overwrites the activations the backward reads.
    bump = dict(batch, last_action=batch["last_action"] + torch.eye(D, device="cuda")[0])
    with torch.no_grad():
        moved = model(bump, state)[0]["policy_logits"] - out["policy_logits"].detach()
    if not use_lstm:
        np.testing.assert_allclose(moved.cpu().numpy(), np.broadcast_to(
            model.policy.weight[:, 513].detach().cpu().numpy(), moved.shape), rtol=1e-3, atol=1e-5)
    else:
        assert moved.abs().max() > 0


@pytest.mark.parametrize("use_lstm", [False, True])
def test_resnet_gaussian_runs_its_entries_at_num_actions_2d(use_lstm):
    """ResNet has no last-action input: a Gaussian(D) net is the int 2D net, bit for bit, forward and backward; the
    action is float32 [T, B, D]."""
    from torchbeast_b200 import nets
    from torchbeast_b200.sampling import ActionSampler
    D, T, B = 5, 3, 4
    gauss = _net("resnet", D, use_lstm, 13)
    flat = nets.ResNet(2 * D, use_lstm)
    flat.load_state_dict(gauss.state_dict())
    batch = _batch("resnet", T - 1, B, D, 14)
    state = _state(gauss, B)
    gauss.action_sampler = ActionSampler(5, 0)
    (a, lg, bg), _ = gauss(dict(batch), state)
    (_, lf, bf), _ = flat(dict(batch), state)
    assert torch.equal(lg, lf) and torch.equal(bg, bf)
    assert a.shape == (T, B, D) and a.dtype == torch.float32
    g = torch.Generator().manual_seed(1)
    gl, gb = torch.randn(lg.shape, generator=g).cuda(), torch.randn(bg.shape, generator=g).cuda()
    for m, (lo, ba) in ((gauss, (lg, bg)), (flat, (lf, bf))):
        m.zero_grad(set_to_none=True)
        ((lo * gl).sum() + (ba * gb).sum()).backward()
    for (n, p), (_, q) in zip(gauss.named_parameters(), flat.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
    gauss.eval()
    with torch.no_grad():
        (a, lg, _), _ = gauss(dict(batch), state)
    assert torch.equal(a, lg[..., :D])


# ---- learning and acting ---------------------------------------------------------------------------------------------


def _opt(model):
    from torchbeast_b200 import optim
    return optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)


@pytest.mark.parametrize("kind", ["atari", "resnet"])
@pytest.mark.parametrize("use_lstm", [False, True])
def test_learn_step_matches_a_torch_reference(kind, use_lstm):
    from tests.test_gaussian_cpu import _torch_loss
    from torchbeast_b200 import learner
    T, B, D = 5, 3, 6
    model = _net(kind, D, use_lstm, 6)
    batch = _batch(kind, T, B, D, 7)
    state = _state(model, B)
    flags = types.SimpleNamespace(**FLAGS)
    out = model.learner_forward(batch, state)
    logits, values = out.policy_logits.cpu().numpy(), out.baseline.cpu().numpy()
    step = learner.learn_step(flags, model, None, batch, state, _opt(model), None, stats_sync=False)
    torch.cuda.synchronize()
    bn = {k: v.cpu().numpy() for k, v in batch.items()}
    d = dict(bl=bn["policy_logits"][1:].astype(np.float64), tl=logits[:-1].astype(np.float64),
             actions=bn["action"][1:].astype(np.float64), rewards=bn["reward"][1:].astype(np.float64),
             done=bn["done"][1:], values=values[:-1].astype(np.float64), bootstrap=values[-1].astype(np.float64),
             weights=np.ones(B))
    want = _torch_loss(d, ent_cost=0.01)
    np.testing.assert_allclose(step["losses"].cpu().numpy(), want["losses"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(step["vtrace"].grad_logits.cpu().numpy()[:-1], want["grad_logits"], rtol=1e-3,
                               atol=1e-5)
    # the header's formulas on the columns: mu gets -adv z exp(-l), l gets adv (1 - z^2) - entropy_cost
    adv = step["vtrace"].pg_advantages.cpu().numpy()
    np.testing.assert_allclose(step["vtrace"].grad_logits.cpu().numpy()[:-1],
                               GO.row_grad(d["tl"], d["actions"], adv, 0.01), rtol=1e-3, atol=1e-5)


@pytest.mark.parametrize("kind", ["atari", "resnet"])
@pytest.mark.parametrize("replay", [None, "uniform", "prioritised"])
def test_learning_eager_equals_graphed(kind, replay):
    from torchbeast_b200 import learner
    from torchbeast_b200.replay import ReplayBuffer
    T, B, steps, D = 8, 4, 6, 6
    batch = _batch(kind, T, B, D, 1)
    runs = []
    for graphed in (False, True):
        model = _net(kind, D, True, 3)
        state = _state(model, B)
        if replay is not None:
            model.replay = ReplayBuffer(6, 2, seed=5, min_size=2, stream_id=0,
                                        priority_exponent=0.6 if replay == "prioritised" else None)
        opt = _opt(model)
        f = types.SimpleNamespace(**FLAGS, cuda_graph=graphed, trust_region_kl=2.0)
        stats = [learner.learn(f, model, None, batch, state, opt, None) for _ in range(steps)]
        runs.append((stats, model.flat_params.cpu().numpy()))
    for s0, s1 in zip(runs[0][0], runs[1][0]):
        for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss", "trust_fraction"):
            assert np.float32(s0[k]).view(np.int32) == np.float32(s1[k]).view(np.int32), k
    assert _bits_equal(runs[0][1], runs[1][1])
    assert np.all(np.isfinite([s["total_loss"] for s in runs[0][0]]))


@pytest.mark.parametrize("prioritised", [False, True])
def test_replay_stores_and_replays_float_action_columns(prioritised):
    """Each fresh column carries a distinct non-integer float tag in action component 0; every replayed column equals,
    leaf for leaf and bit for bit, the stored rollout column its tag names."""
    from torchbeast_b200.replay import ReplayBuffer
    T, B, D = 4, 3, 6
    buf = ReplayBuffer(8, 2, seed=9, min_size=2, stream_id=0, priority_exponent=0.6 if prioritised else None)
    pushed = {}
    for call in range(6):
        b = _batch("atari", T, B, D, 20 + call)
        tag = torch.tensor([call * B + j + 0.125 for j in range(B)], device="cuda")
        b["action"][..., 0] = tag[None, :]
        for j in range(B):
            pushed[float(tag[j])] = {k: v[:, j].clone() for k, v in b.items()}
        if prioritised and buf.priorities is not None:
            buf.priorities.fill_(1.0)
        mixed, _, fresh = buf.mix(b)
        if fresh is None:
            continue
        for j in range(fresh, mixed["action"].shape[1]):
            src = pushed[float(mixed["action"][0, j, 0])]
            for k in src:
                assert torch.equal(mixed[k][:, j], src[k]), k


def test_graphed_actor_matches_the_eager_forward():
    from torchbeast_b200.acting import GraphedActor, bucket_size
    from torchbeast_b200.sampling import ActionSampler
    D, B = 6, 8
    assert bucket_size(B) == B
    model = _net("atari", D, True, 8)
    model.train()
    b = _batch("atari", 0, B, D, 9)
    inputs = {k: b[k] for k in ("frame", "reward", "done", "last_action")}
    state = _state(model, B)
    actor = GraphedActor(model)
    for call in range(3):
        model.action_sampler = ActionSampler(31, 10 * call)
        with torch.no_grad():
            g_out, g_state = actor(inputs, state)
        model.action_sampler = ActionSampler(31, 10 * call)
        with torch.no_grad():
            e_out, e_state = model(inputs, state)
        assert torch.equal(g_out["policy_logits"], e_out["policy_logits"])
        assert g_out["action"].shape == (1, B, D) and g_out["action"].dtype == torch.float32
        assert _bits_equal(g_out["action"].cpu(), e_out["action"].cpu())
        assert all(torch.equal(x, y) for x, y in zip(g_state, e_state))
    model.eval()
    with torch.no_grad():
        out, _ = model(inputs, state)
    assert torch.equal(out["action"], out["policy_logits"][..., :D])


@pytest.mark.parametrize("case", ["upgo", "kickstart", "legal", "teacher", "int_actions"])
def test_continuous_learner_raises_before_anything_is_launched(case):
    from torchbeast_b200 import _lib, learner, nets
    from torchbeast_b200.kickstart import Teacher
    T, B, D = 4, 2, 6
    model = _net("atari", D, False, 1)
    batch = _batch("atari", T, B, D, 1)
    flags = dict(FLAGS)
    if case == "upgo":
        flags["upgo_cost"] = 0.5
    elif case == "kickstart":
        flags["kickstart_cost"] = 0.5
        model.teacher = Teacher(_net("atari", D, False, 2))
    elif case == "legal":
        batch["legal_actions"] = torch.ones(T + 1, B, 2 * D, dtype=torch.bool, device="cuda")
    elif case == "teacher":
        model.teacher = Teacher(nets.AtariNet((4, 84, 84), 2 * D, False))
    else:
        batch["action"] = batch["action"].round().to(torch.int64)
        batch["last_action"] = batch["last_action"].round().to(torch.int64)
    before = model.flat_params.clone()
    launches = _lib.lib().tb_launch_count()
    with pytest.raises(_lib.TorchBeastB200Error, match="not built for a continuous|differs from the learner"):
        learner.learn(types.SimpleNamespace(**flags), model, None, batch, (), _opt(model), None)
    assert _lib.lib().tb_launch_count() == launches
    assert torch.equal(model.flat_params, before)
