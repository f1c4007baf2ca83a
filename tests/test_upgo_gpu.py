"""GPU: the UPGO launch (tb_upgo_loss_f32) against the float64 oracle of tests/upgo_oracle.py on both scan layouts and
every feature group of the loss (hp block, uint8 done, column weights, trust region, PopArt), its bit properties
(a zero cost, beta = +inf, run to run, the total), and learn() with UPGO: eager against graphed for AtariNet and
ResNet with the cost changed between replays, prioritised replay with the trust region, and the step without it.

Rewards, values and the PopArt statistics are multiples of 1/16 (sigma a power of two) and the discount is 0.75 (1/256
for uint8 done, whose discount is (255 - done) * gamma), so every trace switch r + g V' >= V is exact in fp32 and
float64 alike: no row can switch one way in the kernel and the other in the oracle."""
import math
import types

import numpy as np
import pytest
import torch

from tests import trust_region_oracle as TO
from tests import upgo_oracle as UO
from tests.test_replay_gpu import FLAGS, LOSS_KEYS, Learner, _atari, _batch, _collect_graphs, _state  # noqa: F401

pytestmark = pytest.mark.gpu

COSTS = dict(baseline_cost=0.5, entropy_cost=0.01)
GAMMA = {torch.bool: 0.75, torch.uint8: 1.0 / 256}
# (T, B, A): T in {1, 2, 7, 80, 600}, B in {1, 5, 33, 8192}, A in {3, 6, 18} and 11 (no instantiation of its own).
# T = 1, 2 and B = 8192 at T = 1 take the wide layout (one warp per column tile, the whole unroll); the others split T
# over up to 16 warps, whose chunk edges fall on trace switches in about half of the cases.
SHAPES = [(1, 8192, 6), (1, 1, 3), (2, 5, 3), (7, 33, 18), (7, 1, 11), (80, 1, 11), (80, 33, 6), (80, 8192, 3),
          (600, 5, 6), (600, 33, 18)]
# uint8 done (a discount of about 1) only up to T = 80: longer unrolls only grow the return
CASES = [s + (v,) for s in SHAPES for v in ("plain", "hp", "uint8") if v != "uint8" or s[0] <= 80]
LAYOUTS = {"wide": (4, 300), "split": (300, 8)}


def _q(rs, shape, lim=2.0):
    """Multiples of 1/16 in [-lim, lim]."""
    return (np.round(rs.uniform(-lim, lim, size=shape) * 16) / 16).astype(np.float32)


def _inputs(T, B, A, seed, done_dtype=torch.bool):
    rs = np.random.RandomState(seed)
    tl = (1.5 * rs.randn(T, B, A)).astype(np.float32)
    done = rs.rand(T, B) < 0.1
    return dict(behavior_policy_logits=(tl + 0.7 * rs.randn(T, B, A)).astype(np.float32), target_policy_logits=tl,
                actions=rs.randint(0, A, size=(T, B)), rewards=_q(rs, (T, B)),
                done=done if done_dtype == torch.bool else done.astype(np.uint8),
                values=_q(rs, (T, B)), bootstrap_value=_q(rs, (B,)))


def _discounts(kw):
    g = GAMMA[torch.bool if kw["done"].dtype == bool else torch.uint8]
    d = kw["done"]
    return g * ~d if d.dtype == bool else g * (255 - d.astype(np.float64))


def _cuda(kw):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in kw.items()}


def _hp_block(gamma):
    from torchbeast_b200 import learner
    block = torch.zeros(learner.HPARAMS.itemsize, dtype=torch.uint8, device="cuda")
    learner.publish_hparams(learner.pack_hparams(types.SimpleNamespace(**dict(FLAGS, **COSTS, discounting=gamma))), block)
    return block


def _run(kw, upgo_cost=None, hp=False, weights=None, trust_region=None, with_grads=True):
    """One impala_loss_fwd_bwd call on host inputs; returns host arrays (upgo_adv / upgo_loss with UPGO)."""
    from torchbeast_b200 import learner
    d = _cuda(kw)
    gamma = GAMMA[d["done"].dtype]
    extra = dict(upgo_cost=upgo_cost, trust_region=trust_region, with_grads=with_grads)
    if hp:
        extra["hparams_dev"] = _hp_block(gamma)
    if weights is not None:
        extra["column_weights"] = torch.from_numpy(weights).cuda()
    res = learner.impala_loss_fwd_bwd(**d, discounting=gamma, **COSTS, **extra)
    torch.cuda.synchronize()
    res = (res,) if isinstance(res, learner.ImpalaLoss) else res
    host = lambda t: None if t is None else t.cpu().numpy()   # noqa: E731
    out = {k: host(getattr(res[0], k)) for k in res[0]._fields}
    if trust_region is not None:
        out["kl"] = host(res[1].kl)
    if upgo_cost is not None:
        out["upgo_adv"], out["upgo_loss"] = host(res[-1].adv), host(res[-1].loss)
    return out


def _loss_scale(kw, o, cost, weights=None):
    """cost * sum |w (-log pi(a)) adv|: the size of the terms the UPGO loss sums, for its tolerance."""
    lt = TO.log_softmax(np.asarray(kw["target_policy_logits"], np.float64))
    lpa = np.take_along_axis(lt, kw["actions"][..., None], -1)[..., 0]
    w = 1.0 if weights is None else weights[None, :]
    return cost * np.abs(w * lpa * o["adv"]).sum()


def _check_upgo(out, kw, o, cost, weights=None):
    np.testing.assert_allclose(out["upgo_adv"], o["adv"], rtol=1e-4, atol=1e-4)
    assert abs(float(out["upgo_loss"][0]) - o["loss"]) <= 1e-5 * _loss_scale(kw, o, cost, weights) + 1e-6


@pytest.mark.parametrize("T,B,A,variant", CASES)
def test_kernel_matches_float64_oracle(T, B, A, variant):
    seed = 13 * T + B + A
    kw = _inputs(T, B, A, seed, torch.uint8 if variant == "uint8" else torch.bool)
    cost = 0.7
    out = _run(kw, upgo_cost=cost, hp=variant == "hp")
    r, g = np.clip(kw["rewards"], -1, 1), _discounts(kw)
    o = UO.loss(kw["target_policy_logits"], kw["actions"], r, g, kw["values"], kw["bootstrap_value"],
                out["log_rhos"], cost)
    _check_upgo(out, kw, o, cost)
    # grad_logits = the loss's gradient plus UPGO's, against both float64 oracles; row T stays zero
    base = TO.loss(kw["behavior_policy_logits"], kw["target_policy_logits"], kw["actions"], r, g, kw["values"],
                   kw["bootstrap_value"], **COSTS)
    np.testing.assert_allclose(out["grad_logits"][:T], base["grad_logits"] + o["grad_logits"], rtol=1e-4, atol=1e-5)
    assert np.all(out["grad_logits"][T] == 0)
    np.testing.assert_allclose(out["losses"][3], base["losses"][3] + o["loss"], rtol=1e-4,
                               atol=1e-5 * _loss_scale(kw, o, cost) + 1e-4)


def _popart(kw, K, seed):
    """PopArt inputs: head [T+1, B, K] in multiples of 1/16, tasks with column 1 out of range, sigma a power of two."""
    T, B = kw["values"].shape
    rs = np.random.RandomState(seed)
    mu = np.array([0.5, -0.25, 0.0])[:K]
    sigma = np.array([2.0, 0.5, 1.0])[:K]
    task = rs.randint(0, K, size=(T + 1, B))
    task[:, 1] = K
    return dict(values=_q(rs, (T + 1, B, K)), task=task, mu=mu, nu=mu ** 2 + sigma ** 2, sigma=sigma)


def _run_popart(kw, pa, upgo_cost=None, trust_region=None):
    from torchbeast_b200 import learner
    d, p = _cuda(kw), _cuda({k: pa[k] for k in ("values", "task", "mu", "nu")})
    res = learner.impala_loss_popart(d["behavior_policy_logits"], d["target_policy_logits"], d["actions"],
                                     d["rewards"], d["done"], p["values"], p["task"], p["mu"], p["nu"],
                                     discounting=GAMMA[torch.bool], **COSTS, trust_region=trust_region,
                                     upgo_cost=upgo_cost)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in res[0]._asdict().items()}
    out["task_sums"] = res[1].cpu().numpy()
    if trust_region is not None:
        out["kl"] = res[2].kl.cpu().numpy()
    if upgo_cost is not None:
        out["upgo_adv"], out["upgo_loss"] = res[-1].adv.cpu().numpy(), res[-1].loss.cpu().numpy()
    return out


@pytest.mark.parametrize("trust", [False, True])
@pytest.mark.parametrize("variant", ["weighted", "popart1", "popart3"])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("A", [6, 11])
def test_feature_groups_match_float64_oracle(A, layout, variant, trust):
    T, B = LAYOUTS[layout]
    seed = 5 * A + T + len(variant) + trust
    kw = _inputs(T, B, A, seed)
    cost = 1.3
    beta = float(np.float32(np.median(TO.policy_kl(kw["behavior_policy_logits"], kw["target_policy_logits"])))) \
        if trust else None
    r, g = np.clip(kw["rewards"], -1, 1), _discounts(kw)
    if variant == "weighted":
        w = np.random.RandomState(seed).rand(B).astype(np.float32)
        w[2] = 0.0
        off, on = _run(kw, weights=w, trust_region=beta), _run(kw, cost, weights=w, trust_region=beta)
        values, bootstrap, sigma, valid = kw["values"], kw["bootstrap_value"], None, None
    else:
        K = int(variant[-1])
        pa = _popart(kw, K, seed)
        off, on = _run_popart(kw, pa, trust_region=beta), _run_popart(kw, pa, cost, trust_region=beta)
        w = None
        task, ok = pa["task"], pa["task"] < K
        tk = np.where(ok, task, 0)
        v_all = np.where(ok, pa["sigma"][tk] * np.take_along_axis(pa["values"], tk[..., None], -1)[..., 0]
                         + pa["mu"][tk], 0.0)
        values, bootstrap, sigma, valid = v_all[:T], v_all[T], pa["sigma"][tk[:T]], ok[:T]
        assert not valid[:, 1].any() and np.all(on["upgo_adv"][:, 1] == 0)
        assert np.array_equal(off["task_sums"], on["task_sums"])
    mask = None
    if trust:
        mask = on["kl"] <= np.float32(beta)
        assert 0.3 < mask.mean() < 0.7
    o = UO.loss(kw["target_policy_logits"], kw["actions"], r, g, values, bootstrap, on["log_rhos"], cost, mask=mask,
                weights=w, sigma=sigma, valid=valid)
    _check_upgo(on, kw, o, cost, w)
    # UPGO adds its gradient to the loss's and touches nothing else the loss wrote
    np.testing.assert_allclose(on["grad_logits"][:T] - off["grad_logits"][:T], o["grad_logits"], rtol=1e-4, atol=1e-5)
    assert np.array_equal(on["grad_logits"][T], off["grad_logits"][T])
    for k in ("vs", "pg_advantages", "log_rhos", "grad_values"):
        assert np.array_equal(on[k], off[k]), k
    assert np.array_equal(on["losses"][:3], off["losses"][:3])
    want_total = np.float32(np.float64(off["losses"][3]) + np.float64(on["upgo_loss"][0]))
    assert on["losses"][3].view(np.int32) == want_total.view(np.int32)


def _bits(out):
    return {k: v.view(np.int32) for k, v in out.items() if v is not None and v.dtype == np.float32}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_bit_properties(layout):
    T, B = LAYOUTS[layout]
    kw = _inputs(T, B, 6, 21)
    w = np.random.RandomState(3).rand(B).astype(np.float32)
    plain = _run(kw, weights=w)
    # a zero cost leaves every output of the loss launch as it was
    zero = _run(kw, upgo_cost=0.0, weights=w)
    for k, v in _bits(plain).items():
        assert np.array_equal(v, _bits(zero)[k]), k
    assert zero["upgo_loss"][0] == 0.0 and np.any(zero["upgo_adv"] != 0)
    # two runs are bit-identical
    a, b = _run(kw, upgo_cost=0.5, weights=w), _run(kw, upgo_cost=0.5, weights=w)
    for k, v in _bits(a).items():
        assert np.array_equal(v, _bits(b)[k]), k
    # the device-scalar cost gives the float's bits
    c = _run(kw, upgo_cost=torch.tensor([0.5], device="cuda"), weights=w)
    for k, v in _bits(a).items():
        assert np.array_equal(v, _bits(c)[k]), k
    # forward only: no gradient, the same advantage and losses
    f = _run(kw, upgo_cost=0.5, weights=w, with_grads=False)
    assert f["grad_logits"] is None and f["grad_values"] is None
    for k in ("upgo_adv", "upgo_loss", "losses", "vs"):
        assert np.array_equal(f[k].view(np.int32), a[k].view(np.int32)), k
    # beta = +inf gives the bits of UPGO without a trust region
    trust = _run(kw, upgo_cost=0.5, weights=w, trust_region=math.inf)
    for k, v in _bits(a).items():
        assert np.array_equal(v, _bits(trust)[k]), k


def _resnet(num_tasks=None):
    from torchbeast_b200 import polybeast_learner
    m = polybeast_learner.Net(6, True, observation_shape=(3, 64, 64), num_tasks=num_tasks)
    m.reset_parameters_like_torch(seed=3)
    return m


NETS = {
    "atari": (_atari, lambda T, B, k: (_batch(T, B, seed=40 + k), _state(2, B, 512 + 6 + 1, seed=k))),
    "resnet": (_resnet, lambda T, B, k: (_batch(T, B, seed=40 + k, obs=(3, 64, 64)), _state(1, B, 256, seed=k))),
    "resnet_popart": (lambda: _resnet(num_tasks=2),
                      lambda T, B, k: (_batch(T, B, seed=40 + k, obs=(3, 64, 64), num_tasks=2),
                                       _state(1, B, 256, seed=k))),
}


@pytest.mark.parametrize("net", sorted(NETS))
def test_graphed_equals_eager_with_the_cost_changed_between_replays(net):
    make, data = NETS[net]
    runs = {g: Learner(make, graph=g) for g in (False, True)}
    costs = [1.0, 1.0, 0.3, 0.0, 2.5]
    for k, cost in enumerate(costs):
        batch, state = data(4, 4, k)
        for r in runs.values():
            r.flags.upgo_cost = cost
            if net == "resnet_popart":
                r.flags.trust_region_kl = 0.2
        se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
        assert set(se) == set(sg) and "upgo_loss" in se
        for key in LOSS_KEYS + ("upgo_loss",):
            assert se[key] == sg[key], (k, key)
        if cost == 0.0:
            assert se["upgo_loss"] == 0.0
        assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params), k
    assert len(runs[True].model._tb_graphs) == 1   # cost changes captured nothing new
    # turning UPGO off replays another graph and the stats lose its key
    for r in runs.values():
        r.flags.upgo_cost = None
    batch, state = data(4, 4, 99)
    se, sg = runs[False].learn(batch, state), runs[True].learn(batch, state)
    assert "upgo_loss" not in se and "upgo_loss" not in sg
    assert torch.equal(runs[False].model.flat_params, runs[True].model.flat_params)


def test_none_on_a_graph_captured_with_upgo_raises():
    from torchbeast_b200 import learner
    run = Learner(_atari, graph=True)
    run.flags.upgo_cost = 0.5
    batch, state = _batch(4, 4, seed=1), _state(2, 4, 512 + 6 + 1, seed=1)
    run.learn(batch, state)
    (gl,) = run.model._tb_graphs.values()
    run.flags.upgo_cost = None
    with pytest.raises(ValueError, match="UPGO"):
        gl.step(batch, state)
    assert isinstance(gl, learner.GraphedLearner)


def test_prioritised_replay_with_trust_region_and_upgo_matches_the_oracle():
    from torchbeast_b200 import learner
    from torchbeast_b200.replay import Draw, ReplayBuffer
    T, B = 4, 8
    # through learn(): a prioritised buffer, the trust region and UPGO, warm-up and mixing, eager and graphed alike
    runs = {g: Learner(_atari, graph=g, replay=ReplayBuffer(14, 4, seed=8, min_size=4, priority_exponent=0.6))
            for g in (False, True)}
    for k in range(4):
        batch, state = _batch(T, 4, seed=70 + k), _state(2, 4, 512 + 6 + 1, seed=k)
        stats = {}
        for g, r in runs.items():
            r.flags.trust_region_kl, r.flags.upgo_cost = 0.3, 0.8
            stats[g] = r.learn(batch, state)
        for key in LOSS_KEYS + ("upgo_loss", "trust_fraction", "mean_policy_kl"):
            assert stats[False][key] == stats[True][key], (k, key)
        assert torch.equal(runs[False].model.replay.priorities, runs[True].model.replay.priorities)
    # one weighted, trust-region step with a hand-built draw against the oracle on the network's own outputs
    run = Learner(_atari)
    run.flags.trust_region_kl, run.flags.upgo_cost = 0.3, 0.8
    batch, state = _batch(T, B, seed=5), _state(2, B, 512 + 6 + 1, seed=5)
    w = torch.from_numpy(np.random.RandomState(2).rand(B).astype(np.float32)).cuda()
    with torch.no_grad():
        out = run.model.learner_forward(batch, state)
        logits, baseline = out.policy_logits.float().cpu().numpy(), out.baseline.float().cpu().numpy()
    stats = learner.learn_step(run.flags, run.model, run.actor, batch, state, run.opt, None,
                               draw=Draw(None, w, None))
    h = {k: v.cpu().numpy() for k, v in batch.items()}
    bl, tl, act = h["policy_logits"][1:], logits[:-1], h["action"][1:]
    mask = TO.policy_kl(bl, tl) <= 0.3
    assert 0 < mask.mean() <= 1
    lr = TO.loss(bl, tl, act, np.clip(h["reward"][1:], -1, 1), 0.99 * ~h["done"][1:].astype(bool), baseline[:-1],
                 baseline[-1])["log_rhos"]
    o = UO.loss(tl, act, np.clip(h["reward"][1:], -1, 1), 0.99 * ~h["done"][1:].astype(bool), baseline[:-1],
                baseline[-1], lr, 0.8, mask=mask, weights=w.cpu().numpy())
    np.testing.assert_allclose(stats["upgo_loss"], o["loss"], rtol=1e-4, atol=1e-5)
    parts = sum(stats[k] for k in ("pg_loss", "baseline_loss", "entropy_loss", "upgo_loss"))
    np.testing.assert_allclose(stats["total_loss"], parts, rtol=1e-5, atol=1e-6)


def test_without_upgo_the_step_launches_what_it_did():
    from torchbeast_b200 import _lib
    counts, stats = {}, {}
    for name, cost in (("absent", "absent"), ("none", None), ("on", 0.5)):
        run = Learner(_atari)
        if cost != "absent":
            run.flags.upgo_cost = cost
        batch, state = _batch(4, 4, seed=9), _state(2, 4, 512 + 6 + 1, seed=9)
        run.learn(batch, state)            # first step: one-time set-up launches
        before = _lib.lib().tb_launch_count()
        stats[name] = run.learn(batch, state)
        counts[name] = _lib.lib().tb_launch_count() - before
    assert counts["none"] == counts["absent"] and counts["on"] == counts["absent"] + 1
    assert "upgo_loss" not in stats["absent"] and "upgo_loss" not in stats["none"]
    assert "upgo_loss" in stats["on"]


def test_invalid_cost_raises_before_any_launch():
    from torchbeast_b200 import _lib
    for graph in (False, True):
        run = Learner(_atari, graph=graph)
        run.flags.upgo_cost = math.nan
        before = _lib.lib().tb_launch_count()
        params = run.model.flat_params.clone()
        with pytest.raises(ValueError, match="upgo_cost"):
            run.learn(_batch(4, 4, seed=1), _state(2, 4, 512 + 6 + 1, seed=1))
        assert _lib.lib().tb_launch_count() == before and torch.equal(params, run.model.flat_params)
