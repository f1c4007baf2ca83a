"""GPU: the trust-region loss kernels against the float64 oracle of tests/trust_region_oracle.py on both scan layouts,
their limits (beta = +inf, identical policies at beta = 0) against the existing entry points bit for bit, run-to-run
determinism, and learn() with the trust region: eager against graphed with beta changed between replays, with uniform
and prioritised replay, and with PopArt."""
import math
import types

import numpy as np
import pytest
import torch

from tests import trust_region_oracle as TO
from tests.test_replay_gpu import FLAGS, LOSS_KEYS, Learner, _atari, _batch, _collect_graphs, _state  # noqa: F401

pytestmark = pytest.mark.gpu

# (T, B): T = 4 leaves one time step chunk per warp, so the kernel takes the wide layout (one warp per column tile, the
# whole unroll); T = 300 on 8 columns splits T over 16 warps (pass 1 forms the affine maps and writes kl)
LAYOUTS = {"wide": (4, 300), "split": (300, 8)}
COSTS = dict(discounting=0.99, baseline_cost=0.5, entropy_cost=0.01)
# kl in fp32 against float64: |kl - kl64| <= KL_ATOL + KL_RTOL * kl64
KL_ATOL, KL_RTOL = 1e-5, 1e-4


def _inputs(T, B, A, seed, same_logits=False):
    rs = np.random.RandomState(seed)
    tl = (1.5 * rs.randn(T, B, A)).astype(np.float32)
    bl = tl.copy() if same_logits else (tl + 0.7 * rs.randn(T, B, A)).astype(np.float32)
    return dict(behavior_policy_logits=bl, target_policy_logits=tl, actions=rs.randint(0, A, size=(T, B)),
                rewards=(2 * rs.randn(T, B)).astype(np.float32), done=rs.rand(T, B) < 0.1,
                values=rs.randn(T, B).astype(np.float32), bootstrap_value=rs.randn(B).astype(np.float32))


def _cuda(kw):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in kw.items() if not k.startswith("_")}


def _hp_block():
    from torchbeast_b200 import learner
    block = torch.zeros(learner.HPARAMS.itemsize, dtype=torch.uint8, device="cuda")
    learner.publish_hparams(learner.pack_hparams(types.SimpleNamespace(**dict(FLAGS, **COSTS))), block)
    return block


def _popart_args(kw, K=1, identity=True, seed=0):
    """PopArt inputs on the same rows: the value head [T+1, B, K] with the bootstrap row, tasks and statistics.  With
    `identity` (K = 1, mu = 0, nu = 1: sigma = 1) the PopArt loss is the plain one."""
    T, B = kw["values"].shape
    rs = np.random.RandomState(seed)
    head = rs.randn(T + 1, B, K).astype(np.float32)
    task = rs.randint(0, K, size=(T + 1, B))
    if identity:
        head[:T, :, 0], head[T, :, 0] = kw["values"], kw["bootstrap_value"]
        mu, nu = np.zeros(K), np.ones(K)
    else:
        mu = rs.randn(K)
        nu = mu ** 2 + rs.rand(K) + 0.5
    return dict(values=head, task=task, mu=mu, nu=nu)


def _run(kw, variant, trust_region=None):
    """One loss call of `variant` (plain, hp, weighted, popart) on host inputs; returns host arrays."""
    from torchbeast_b200 import learner
    d = _cuda(kw)
    extra = {} if trust_region is None else dict(trust_region=trust_region)
    if variant == "popart":
        pa = _cuda(kw["_popart"])
        res = learner.impala_loss_popart(d["behavior_policy_logits"], d["target_policy_logits"], d["actions"],
                                         d["rewards"], d["done"], pa["values"], pa["task"], pa["mu"], pa["nu"],
                                         **COSTS, **extra)
        loss, sums = res[0], res[1]
        trust = res[2] if trust_region is not None else None
    else:
        args = d
        if variant == "hp":
            extra["hparams_dev"] = _hp_block()
        if variant == "weighted":
            extra["column_weights"] = torch.from_numpy(kw["_weights"]).cuda()
        res = learner.impala_loss_fwd_bwd(**args, **COSTS, **extra)
        loss, trust = (res, None) if trust_region is None else res
        sums = None
    torch.cuda.synchronize()
    host = lambda t: None if t is None else t.cpu().numpy()   # noqa: E731
    out = {k: host(getattr(loss, k)) for k in loss._fields}
    if trust is not None:
        out["kl"], out["trust_out"] = host(trust.kl), host(trust.sums)
    if sums is not None:
        out["task_sums"] = host(sums)
    return out


def _with_variant(kw, variant, B, seed):
    kw = dict(kw)
    if variant == "weighted":
        w = np.random.RandomState(seed).rand(B).astype(np.float32)
        w[1] = 0.0
        kw["_weights"] = w
    if variant == "popart":
        kw["_popart"] = _popart_args(kw)
    return kw


@pytest.mark.parametrize("variant", ["plain", "hp", "weighted", "popart"])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("A", [3, 6, 18, 11])       # 11: no instantiation of its own, the generic-A kernel
def test_kernel_matches_float64_oracle(A, layout, variant):
    T, B = LAYOUTS[layout]
    seed = 7 * A + T
    kw = _with_variant(_inputs(T, B, A, seed), variant, B, seed)
    kl64 = TO.policy_kl(kw["behavior_policy_logits"], kw["target_policy_logits"])
    beta = float(np.float32(np.median(kl64)))                        # about half the rows untrusted
    out = _run(kw, variant, trust_region=beta)
    # kl against float64
    assert np.all(np.abs(out["kl"] - kl64) <= KL_ATOL + KL_RTOL * kl64)
    mask = out["kl"] <= np.float32(beta)                             # the kernel's own mask
    assert 0.3 < mask.mean() < 0.7
    o = TO.loss(kw["behavior_policy_logits"], kw["target_policy_logits"], kw["actions"],
                np.clip(kw["rewards"], -1, 1), 0.99 * ~kw["done"], kw["values"], kw["bootstrap_value"], mask=mask,
                baseline_cost=COSTS["baseline_cost"], entropy_cost=COSTS["entropy_cost"], weights=kw.get("_weights"))
    assert out["trust_out"][0] == o["trusted"]
    np.testing.assert_allclose(out["trust_out"][1], o["kl_sum"], rtol=1e-4)
    for k in ("log_rhos", "behavior_action_log_probs", "target_action_log_probs"):
        np.testing.assert_allclose(out[k], o[{"log_rhos": "log_rhos", "behavior_action_log_probs": "behavior_alp",
                                              "target_action_log_probs": "target_alp"}[k]], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(out["vs"], o["vs"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(out["pg_advantages"], o["pg_adv"], rtol=1e-4, atol=1e-4)
    assert np.all(out["pg_advantages"][~mask] == 0)
    np.testing.assert_allclose(out["losses"], o["losses"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(out["grad_logits"][:T], o["grad_logits"], rtol=1e-4, atol=1e-5)
    assert np.all(out["grad_logits"][T] == 0)
    gv = out["grad_values"][:T, :, 0] if variant == "popart" else out["grad_values"][:T]
    np.testing.assert_allclose(gv, o["grad_values"], rtol=1e-4, atol=1e-5)


def _bits(out):
    return {k: v.view(np.int32) for k, v in out.items() if v is not None and v.dtype == np.float32}


@pytest.mark.parametrize("variant", ["plain", "hp", "weighted", "popart"])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("A", [6, 11])
def test_limits_are_bit_identical_to_the_existing_entry_points(A, layout, variant):
    T, B = LAYOUTS[layout]
    seed = 3 * A + B
    kw = _with_variant(_inputs(T, B, A, seed), variant, B, seed)
    if variant == "popart":
        kw["_popart"] = _popart_args(kw, K=3, identity=False, seed=seed)
    plain = _run(kw, variant)
    for beta in (math.inf, torch.tensor([math.inf], device="cuda")):
        trust = _run(kw, variant, trust_region=beta)
        assert trust["trust_out"][0] == T * B
        for k, v in _bits(plain).items():
            assert np.array_equal(v, _bits(trust)[k]), k
        if variant == "popart":
            assert np.array_equal(plain["task_sums"], trust["task_sums"])
    # identical policies: kl = 0 exactly, trusted at beta = 0
    same = _with_variant(_inputs(T, B, A, seed, same_logits=True), variant, B, seed)
    if variant == "popart":
        same["_popart"] = kw["_popart"]
    plain, trust = _run(same, variant), _run(same, variant, trust_region=0.0)
    assert np.all(trust["kl"] == 0) and trust["trust_out"].tolist() == [T * B, 0.0]
    for k, v in _bits(plain).items():
        assert np.array_equal(v, _bits(trust)[k]), k


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_two_runs_are_bit_identical(layout):
    T, B = LAYOUTS[layout]
    kw = _with_variant(_inputs(T, B, 6, 11), "weighted", B, 11)
    beta = float(np.median(TO.policy_kl(kw["behavior_policy_logits"], kw["target_policy_logits"])))
    a, b = _run(kw, "weighted", beta), _run(kw, "weighted", beta)
    for k, v in _bits(a).items():
        assert np.array_equal(v, _bits(b)[k]), k
    assert "trust_out" in _bits(a)


def test_untrusted_row_never_counts_nan_kl():
    T, B, A = 6, 40, 6
    kw = _inputs(T, B, A, 5)
    kw["behavior_policy_logits"][2, 3, 1] = np.nan
    out = _run(kw, "plain", trust_region=math.inf)
    assert np.isnan(out["kl"][2, 3]) and out["trust_out"][0] == T * B - 1 and np.isnan(out["trust_out"][1])
    assert out["pg_advantages"][2, 3] == 0


def _replay(kind):
    from torchbeast_b200.replay import ReplayBuffer
    if kind == "uniform":
        return ReplayBuffer(14, 6, seed=8, min_size=8)
    return ReplayBuffer(14, 6, seed=8, min_size=8, priority_exponent=0.6, importance_exponent=0.4)


@pytest.mark.parametrize("replay", [None, "uniform", "prioritized"])
def test_graphed_equals_eager_with_beta_changed_between_replays(replay):
    T, Bf = 4, 4
    runs = {g: Learner(_atari, graph=g, replay=None if replay is None else _replay(replay)) for g in (False, True)}
    betas = [0.5, 0.5, 0.05, math.inf, 0.0, 0.2, 1e30]
    for k, beta in enumerate(betas):
        batch, state = _batch(T, Bf, seed=60 + k), _state(2, Bf, 512 + 6 + 1, seed=k)
        for r in runs.values():
            r.flags.trust_region_kl = beta
        se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
        for key in LOSS_KEYS + ("trust_fraction", "mean_policy_kl"):
            assert se[key] == sg[key], (k, key)
        assert 0.0 <= se["trust_fraction"] <= 1.0
        if beta == math.inf:
            assert se["trust_fraction"] == 1.0
        assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params), k
        if replay == "prioritized":
            assert torch.equal(runs[False].model.replay.priorities, runs[True].model.replay.priorities)
    # one graph per replay phase; beta changes captured nothing new
    assert len(runs[True].model._tb_graphs) == (1 if replay is None else 2)
    # turning the trust region off replays another graph, and the stats lose its keys
    for r in runs.values():
        r.flags.trust_region_kl = None
    batch, state = _batch(T, Bf, seed=99), _state(2, Bf, 512 + 6 + 1, seed=99)
    se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
    assert "trust_fraction" not in se and "trust_fraction" not in sg
    assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params)


def test_infinite_beta_learns_like_no_trust_region():
    T, Bf = 4, 4
    plain, trust = Learner(_atari), Learner(_atari)
    trust.flags.trust_region_kl = math.inf
    for k in range(2):
        batch, state = _batch(T, Bf, seed=30 + k), _state(2, Bf, 512 + 6 + 1, seed=k)
        sp, st = plain.learn(batch, state), trust.learn(batch, state)
        assert set(st) - set(sp) == {"trust_fraction", "mean_policy_kl"}
        assert all(sp[key] == st[key] for key in LOSS_KEYS)
        assert st["trust_fraction"] == 1.0 and st["mean_policy_kl"] > 0
        assert torch.equal(plain.model.flat_params, trust.model.flat_params)


@pytest.mark.parametrize("graph", [False, True])
def test_popart_with_trust_region_through_learn(graph):
    from torchbeast_b200 import polybeast_learner

    def make():
        m = polybeast_learner.Net(6, True, observation_shape=(3, 64, 64), num_tasks=2)
        m.reset_parameters_like_torch(seed=3)
        return m
    runs = {g: Learner(make, graph=g) for g in (False, graph)}
    for k, beta in enumerate((0.3, 0.03, math.inf)):
        batch, state = _batch(4, 4, seed=1 + k, obs=(3, 64, 64), num_tasks=2), _state(1, 4, 256, seed=k)
        stats = {}
        for g, r in runs.items():
            r.flags.trust_region_kl = beta
            stats[g] = r.learn(batch, state)
        s = stats[graph]
        assert "popart_mu" in s and 0.0 <= s["trust_fraction"] <= 1.0 and s["mean_policy_kl"] >= 0
        if beta == math.inf:
            assert s["trust_fraction"] == 1.0
        for key in LOSS_KEYS + ("trust_fraction", "mean_policy_kl", "popart_mu", "popart_sigma"):
            assert stats[False][key] == s[key], (k, key)
        assert torch.equal(runs[False].model.flat_params, runs[graph].model.flat_params)


def test_invalid_flag_raises_before_any_launch():
    from torchbeast_b200 import _lib
    run = Learner(_atari)
    run.flags.trust_region_kl = -0.1
    before = _lib.lib().tb_launch_count()
    params = run.model.flat_params.clone()
    with pytest.raises(ValueError, match="trust_region_kl"):
        run.learn(_batch(4, 4, seed=1), _state(2, 4, 512 + 6 + 1, seed=1))
    assert _lib.lib().tb_launch_count() == before and torch.equal(params, run.model.flat_params)
