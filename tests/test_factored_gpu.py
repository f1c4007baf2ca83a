"""GPU: factored (multi-discrete) action spaces.  tb_impala_loss_factored_f32 against the float64 oracle of
tests/factored_oracle.py on every feature path and both launch layouts; D = 1 and size-1 padding components against
the flat kernel, bit for bit; the factored sampler against the oracle's Philox rule, D = 1 against
tb_sample_actions_f32, and eager against graphed; AtariNet and ResNet learning eager and graphed, with uniform and
prioritised replay; a factored GraphedActor call against the eager forward; and the four cases that raise."""
import gc
import types

import numpy as np
import pytest
import torch

from tests import factored_oracle as FO

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


def _inputs(T, B, dims, seed, K=None):
    rs = np.random.RandomState(seed)
    A = sum(dims)
    d = dict(bl=(2 * rs.randn(T, B, A)).astype(np.float32), tl=(2 * rs.randn(T, B, A)).astype(np.float32),
             actions=np.stack([rs.randint(0, a, size=(T, B)) for a in dims], -1).astype(np.int64),
             rewards=(2 * rs.randn(T, B)).astype(np.float32), done=rs.rand(T, B) < 0.1,
             values=rs.randn(T, B).astype(np.float32), bootstrap=rs.randn(B).astype(np.float32),
             weights=rs.rand(B).astype(np.float32))
    if K is not None:
        d["n"] = rs.randn(T + 1, B, K).astype(np.float32)
        d["task"] = rs.randint(0, K, size=(T + 1, B)).astype(np.int64)
        d["mu"] = 0.3 * rs.randn(K)
        d["nu"] = d["mu"] ** 2 + 0.5 + rs.rand(K)
    return d


def _cu(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _run(d, dims, path, actions=None, flat=False):
    """One loss call through learner.impala_loss_fwd_bwd / impala_loss_popart; flat: the flat entry point on the same
    logits (actions [T, B])."""
    from torchbeast_b200 import learner
    acts = d["actions"] if actions is None else actions
    kw = dict(discounting=0.99, baseline_cost=0.5, entropy_cost=0.01)
    space = None if flat else dims
    beta = 0.8 if "trust" in path else None
    hp = None
    if "hp" in path:
        rec = learner.pack_hparams(types.SimpleNamespace(grad_norm_clipping=None, reward_clipping="abs_one", **kw))
        hp = torch.zeros(learner.HPARAMS.itemsize, dtype=torch.uint8, device="cuda")
        learner.publish_hparams(rec, hp)
    if "popart" in path:
        res = learner.impala_loss_popart(_cu(d["bl"]), _cu(d["tl"]), _cu(acts), _cu(d["rewards"]), _cu(d["done"]),
                                         _cu(d["n"]), _cu(d["task"]), _cu(d["mu"]), _cu(d["nu"]), hparams_dev=hp,
                                         trust_region=beta, action_space=space, **kw)
        loss, sums = res[0], res[1]
        trust = res[2] if beta is not None else None
    else:
        res = learner.impala_loss_fwd_bwd(
            _cu(d["bl"]), _cu(d["tl"]), _cu(acts), _cu(d["rewards"]), _cu(d["done"]), _cu(d["values"]),
            _cu(d["bootstrap"]), hparams_dev=hp, trust_region=beta, action_space=space,
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


def _oracle(d, dims, path):
    kw = dict(entropy_cost=0.01, trust_beta=0.8 if "trust" in path else None,
              weights=d["weights"] if "weighted" in path else None)
    if "popart" in path:
        return FO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], d["n"], None, dims,
                              popart=(d["task"], d["mu"], d["nu"]), **kw)
    return FO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], d["values"], d["bootstrap"], dims,
                          **kw)


PATHS = ["plain", "hp", "weighted", "trust", "weighted_trust", "popart", "popart_trust"]
SPACES = [(3, 3, 2), (2, 1, 5, 1, 4, 3, 1)]


@pytest.mark.parametrize("dims", SPACES)
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("T,B", [(80, 32), (4, 64)])  # split-T layout; single-launch layout (T <= 4)
def test_loss_matches_the_oracle(dims, path, T, B):
    d = _inputs(T, B, dims, 100 + T + len(dims), K=3 if "popart" in path else None)
    got, want = _run(d, dims, path), _oracle(d, dims, path)
    tol = dict(rtol=2e-4, atol=2e-4)
    for k in ("vs", "pg_advantages", "log_rhos", "target_action_log_probs", "behavior_action_log_probs"):
        wk = {"pg_advantages": "pg_adv", "target_action_log_probs": "target_alp",
              "behavior_action_log_probs": "behavior_alp"}.get(k, k)
        np.testing.assert_allclose(got[k], want[wk], err_msg=k, **tol)
    np.testing.assert_allclose(got["losses"], want["losses"], rtol=2e-4, atol=1e-3)
    np.testing.assert_allclose(got["grad_logits"][:-1], want["grad_logits"], rtol=1e-3, atol=1e-5)
    assert np.all(got["grad_logits"][-1] == 0)
    gv = got["grad_values"]
    np.testing.assert_allclose(gv if "popart" in path else gv[:-1], want["grad_values"], rtol=1e-3, atol=1e-5)
    if "trust" in path:
        np.testing.assert_allclose(got["kl"], want["kl"], rtol=1e-4, atol=1e-5)
        assert got["trust_out"][0] == want["trusted"]
    if "popart" in path:
        np.testing.assert_allclose(got["task_sums"], want["task_sums"], rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("A", [6, 11])  # a static-A and a dynamic-A flat kernel
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("T,B", [(80, 32), (4, 64)])
def test_one_component_gives_the_flat_bits(A, path, T, B):
    d = _inputs(T, B, (A,), 7 + A, K=3 if "popart" in path else None)
    fac, flat = _run(d, (A,), path), _run(d, (A,), path, actions=d["actions"][..., 0], flat=True)
    assert fac.keys() == flat.keys()
    for k in fac:
        assert _bits_equal(fac[k], flat[k]) if fac[k].dtype != np.float64 else np.array_equal(fac[k], flat[k]), k


@pytest.mark.parametrize("A", [6, 11])
@pytest.mark.parametrize("path", ["plain", "weighted_trust", "popart"])
def test_size_one_components_around_one_give_the_flat_bits(A, path):
    T, B = 80, 32
    d = _inputs(T, B, (A,), 30 + A, K=3 if "popart" in path else None)
    flat = _run(d, (A,), path, actions=d["actions"][..., 0], flat=True)
    rs = np.random.RandomState(4)
    dims = (1, 1, A, 1)
    pad = lambda x: np.concatenate([rs.randn(T, B, 2).astype(np.float32), x, rs.randn(T, B, 1).astype(np.float32)], -1)
    e = dict(d, bl=pad(d["bl"]), tl=pad(d["tl"]),
             actions=np.concatenate([np.zeros((T, B, 2), np.int64), d["actions"], np.zeros((T, B, 1), np.int64)], -1))
    fac = _run(e, dims, path)
    for k in flat:
        if k == "grad_logits":
            assert _bits_equal(fac[k][..., 2:2 + A], flat[k]), k
            assert np.all(fac[k][..., [0, 1, A + 2]] == 0)
        elif flat[k].dtype == np.float64:
            assert np.array_equal(fac[k], flat[k]), k
        else:
            assert _bits_equal(fac[k], flat[k]), k


def test_out_of_range_component_poisons_its_row():
    d = _inputs(6, 4, (3, 2), 3)
    acts = d["actions"].copy()
    acts[2, 1, 1] = 2
    got = _run(d, (3, 2), "plain", actions=acts)
    assert np.isnan(got["target_action_log_probs"][2, 1]) and np.isnan(got["losses"][3])
    t = got["target_action_log_probs"].copy()
    t[2, 1] = 0
    assert np.isfinite(t).all()


# ---- sampling --------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("dims", [(3, 3, 2), (2, 1, 5, 1, 4, 3, 1), tuple(range(1, 17)), (18,)])
def test_sampler_matches_the_oracle(dims):
    from torchbeast_b200.sampling import ActionSampler
    T, B = 3, 257
    x = (3 * np.random.RandomState(len(dims)).randn(T, B, sum(dims))).astype(np.float32)
    x[0, 0, :] = np.nan                                  # every segment of this row: -1
    s = ActionSampler(2 ** 33 + 5, 17)
    got = s.sample(_cu(x), action_dims=dims).cpu().numpy()
    assert s.step == 17 + T and got.shape == (T, B, len(dims))
    want, margin = FO.sample_actions(x, dims, 2 ** 33 + 5, 17)
    from oracle import sampling_np as SO
    ok = margin >= np.array([SO.margin_threshold(a) for a in dims])
    assert np.array_equal(got[ok], want[ok]) and ok.mean() > 0.95
    assert np.all(got[0, 0] == -1)
    assert np.all((got[1:] >= 0) & (got[1:] < np.array(dims)))


def test_one_component_sampler_gives_the_flat_actions_and_graphed_equals_eager():
    from torchbeast_b200 import _lib
    from torchbeast_b200.sampling import ActionSampler, sample_factored
    T, B, A = 4, 300, 7
    x = _cu((3 * np.random.RandomState(1).randn(T, B, A)).astype(np.float32))
    ids = torch.arange(B, dtype=torch.int64, device="cuda") * 7 - 100
    flat = ActionSampler(99, 5).sample(x, ids)
    fac = ActionSampler(99, 5).sample(x, ids, action_dims=(A,))
    assert torch.equal(fac[..., 0], flat)
    # the device (seed, step) form, captured in a graph, gives the host form's actions at every replayed step
    dims = (3, 1, 2, 1)
    y = _cu((3 * np.random.RandomState(2).randn(1, B, sum(dims))).astype(np.float32))
    seed_step = torch.zeros(2, dtype=torch.int64, device="cuda")
    sample_factored(y, dims, ids, seed_step=seed_step)                    # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = sample_factored(y, dims, ids, seed_step=seed_step)
    for step in (0, 1, 12345):
        seed_step.copy_(torch.tensor([2 ** 40 + 3, step]))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, sample_factored(y, dims, ids, seed=2 ** 40 + 3, step=step))
    assert _lib.lib().tb_launch_count() > 0


# ---- nets, acting and learning --------------------------------------------------------------------------------------

DIMS = (3, 3, 2)


def _net(kind, dims, use_lstm, seed):
    from torchbeast_b200 import nets
    m = nets.AtariNet((4, 84, 84), dims, use_lstm) if kind == "atari" else nets.ResNet(dims, use_lstm)
    m.reset_parameters_like_torch(seed=seed)
    return m


def _batch(kind, T, B, dims, seed):
    """A small synthetic task: reward 1 when component 0's action is 0, else 0, so the loss can fall."""
    g = torch.Generator().manual_seed(seed)
    D = len(dims)
    action = torch.stack([torch.randint(0, a, (T + 1, B), generator=g) for a in dims], -1)
    b = dict(frame=torch.randint(0, 255, (T + 1, B, 4, 84, 84), generator=g, dtype=torch.uint8),
             reward=(action[..., 0] == 0).float(), done=torch.rand(T + 1, B, generator=g) < 0.1,
             episode_return=torch.randn(T + 1, B, generator=g), policy_logits=torch.randn(T + 1, B, sum(dims), generator=g),
             action=action)
    if kind == "atari":
        b["last_action"] = torch.cat([torch.zeros(1, B, D, dtype=torch.int64), action[:-1]])
    return {k: v.cuda() for k, v in b.items()}


def _state(model, B):
    g = torch.Generator().manual_seed(B)
    return tuple((0.1 * torch.randn(s.shape, generator=g)).cuda() for s in model.initial_state(B))


def _opt(model):
    from torchbeast_b200 import optim
    return optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)


@pytest.mark.parametrize("kind", ["atari", "resnet"])
@pytest.mark.parametrize("replay", [None, "uniform", "prioritised"])
def test_learning_eager_equals_graphed_and_the_loss_falls(kind, replay):
    from torchbeast_b200 import learner
    from torchbeast_b200.replay import ReplayBuffer
    T, B, steps = 8, 4, 12
    batch = _batch(kind, T, B, DIMS, 1)
    batch["frame"].zero_()  # one observation: the value and the policy can fit the task within a few steps
    runs = []
    for graphed in (False, True):
        model = _net(kind, DIMS, True, 3)
        state = _state(model, B)
        if replay is not None:
            model.replay = ReplayBuffer(6, 2, seed=5, min_size=2, stream_id=0,
                                        priority_exponent=0.6 if replay == "prioritised" else None)
        opt = _opt(model)
        f = types.SimpleNamespace(**FLAGS, cuda_graph=graphed, trust_region_kl=5.0)
        stats = [learner.learn(f, model, None, batch, state, opt, None) for _ in range(steps)]
        runs.append((stats, model.flat_params.cpu().numpy()))
    for s0, s1 in zip(runs[0][0], runs[1][0]):
        for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss", "trust_fraction"):
            assert np.float32(s0[k]).view(np.int32) == np.float32(s1[k]).view(np.int32), k
    assert _bits_equal(runs[0][1], runs[1][1])
    tot = [s["total_loss"] for s in runs[0][0]]
    assert np.all(np.isfinite(tot))
    assert np.mean(tot[-3:]) < np.mean(tot[:3])


@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_learning_with_popart_trust_region_and_hparam_changes_eager_equals_graphed(kind):
    from torchbeast_b200 import learner, nets
    T, B = 6, 4
    batch = _batch(kind, T, B, DIMS, 2)
    runs = []
    for graphed in (False, True):
        model = (nets.AtariNet((4, 84, 84), DIMS, False, num_tasks=1) if kind == "atari"
                 else nets.ResNet(DIMS, False, num_tasks=1))
        model.reset_parameters_like_torch(seed=4)
        opt = _opt(model)
        stats = []
        for i in range(4):  # the loss hyper-parameters change between replays
            f = types.SimpleNamespace(**dict(FLAGS, entropy_cost=0.01 * (i + 1), discounting=0.99 - 0.01 * i,
                                             baseline_cost=0.5 + 0.1 * i), cuda_graph=graphed, trust_region_kl=1.0)
            stats.append(learner.learn(f, model, None, batch, (), opt, None))
        runs.append((stats, model.flat_params.cpu().numpy()))
    for s0, s1 in zip(runs[0][0], runs[1][0]):
        assert np.float32(s0["total_loss"]).view(np.int32) == np.float32(s1["total_loss"]).view(np.int32)
    assert _bits_equal(runs[0][1], runs[1][1])


def test_learn_step_loss_matches_the_oracle_and_the_k_hot_reaches_the_core():
    from torchbeast_b200 import learner
    T, B = 5, 3
    model = _net("atari", DIMS, False, 6)
    batch = _batch("atari", T, B, DIMS, 7)
    flags = types.SimpleNamespace(**FLAGS)
    out = model.learner_forward(batch, ())
    logits, values = out.policy_logits.cpu().numpy(), out.baseline.cpu().numpy()
    step = learner.learn_step(flags, model, None, batch, (), _opt(model), None, stats_sync=False)
    torch.cuda.synchronize()
    bn = {k: v.cpu().numpy() for k, v in batch.items()}
    want = FO.impala_loss(bn["policy_logits"][1:], logits[:-1], bn["action"][1:], bn["reward"][1:], bn["done"][1:],
                          values[:-1], values[-1], DIMS, entropy_cost=0.01)
    np.testing.assert_allclose(step["losses"].cpu().numpy(), want["losses"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(step["vtrace"].grad_logits.cpu().numpy()[:-1], want["grad_logits"], rtol=1e-3,
                               atol=1e-5)
    # the K-hot: a different last action changes the logits; the one-hot of the flat space is not what is read
    other = dict(batch, last_action=(batch["last_action"] + 1) % torch.tensor(DIMS, device="cuda"))
    assert not torch.equal(model.learner_forward(other, ()).policy_logits, model.learner_forward(batch, ()).policy_logits)


@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_graphed_actor_matches_the_eager_forward(kind):
    from torchbeast_b200.acting import GraphedActor
    from torchbeast_b200.sampling import ActionSampler
    model = _net(kind, DIMS, True, 8)
    model.train()
    B = 5
    b = _batch(kind, 0, B, DIMS, 9)
    names = ("frame", "reward", "done") + (("last_action",) if kind == "atari" else ())
    inputs = {k: b[k] for k in names}
    state = _state(model, B)
    actor = GraphedActor(model)
    for call in range(3):
        model.action_sampler = ActionSampler(31, 10 * call)
        with torch.no_grad():
            g_out, g_state = actor(inputs, state)
        model.action_sampler = ActionSampler(31, 10 * call)
        with torch.no_grad():
            e_out, e_state = model(inputs, state)
        if kind == "atari":
            g_act, e_act = g_out["action"], e_out["action"]
            assert torch.equal(g_out["policy_logits"], e_out["policy_logits"])
        else:
            g_act, e_act = g_out[0], e_out[0]
            assert torch.equal(g_out[1], e_out[1])
        assert g_act.shape == (1, B, len(DIMS)) and torch.equal(g_act, e_act)
        assert all(torch.equal(x, y) for x, y in zip(g_state, e_state))
    model.eval()
    with torch.no_grad():
        out, _ = model(inputs, state)
    logits = out["policy_logits"] if kind == "atari" else out[1]
    act = out["action"] if kind == "atari" else out[0]
    want = torch.stack([s.argmax(-1) for s in logits.split(DIMS, -1)], -1)
    assert torch.equal(act, want)


@pytest.mark.parametrize("case", ["upgo", "kickstart", "legal", "teacher"])
def test_factored_learner_raises_before_anything_is_launched(case):
    from torchbeast_b200 import _lib, learner
    from torchbeast_b200.kickstart import Teacher
    T, B = 4, 2
    model = _net("atari", DIMS, False, 1)
    batch = _batch("atari", T, B, DIMS, 1)
    flags = dict(FLAGS)
    if case == "upgo":
        flags["upgo_cost"] = 0.5
    elif case == "kickstart":
        flags["kickstart_cost"] = 0.5
        model.teacher = Teacher(_net("atari", DIMS, False, 2))
    elif case == "legal":
        batch["legal_actions"] = torch.ones(T + 1, B, sum(DIMS), dtype=torch.bool, device="cuda")
    else:
        model.teacher = Teacher(_net("atari", (4, 4), False, 2))
    before = model.flat_params.clone()
    launches = _lib.lib().tb_launch_count()
    with pytest.raises(_lib.TorchBeastB200Error, match="not built for a factored|differs from the learner"):
        learner.learn(types.SimpleNamespace(**flags), model, None, batch, (), _opt(model), None)
    assert _lib.lib().tb_launch_count() == launches
    assert torch.equal(model.flat_params, before)
