"""GPU: PopArt value normalisation.  With one task, identity statistics and beta = 0 a learn step is bit-identical to
the same model without PopArt; the loss and update kernels against the float64 restatement (tests/popart_oracle.py)
at four tasks, on both scan layouts and the hyper-parameter block path; determinism; graph replay against eager with
beta and the task mix changed between steps; out-of-range task ids; the acting graph."""
import gc
import types

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests import popart_oracle as PO

pytestmark = pytest.mark.gpu

A = 6
FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


@pytest.fixture(autouse=True)
def _collect_graphs():
    yield
    gc.collect()
    torch.cuda.synchronize()


def _make(net, use_lstm, precision, **kw):
    from torchbeast_b200 import nets
    if net == "atari":
        m = nets.AtariNet((4, 84, 84), A, use_lstm, precision=precision, **kw)
    else:
        m = nets.ResNet(A, use_lstm, precision=precision, **kw)
    m.reset_parameters_like_torch(seed=5)
    return m


def _state(m, B):
    return tuple(s.clone() for s in m.initial_state(B))


def _batch(T, B, net, seed):
    return {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=seed, with_last_action=(net == "atari")).items()}


IDENTITY_CASES = [("atari", lstm, T, B) for lstm in (False, True) for T, B in ((4, 2), (80, 32))] + \
                 [("resnet", lstm, 4, 2) for lstm in (False, True)]


@pytest.mark.parametrize("precision", [None, "fp32"])
@pytest.mark.parametrize("net,use_lstm,T,B", IDENTITY_CASES)
def test_identity_step_is_bit_identical(net, use_lstm, T, B, precision):
    from torchbeast_b200 import learner, optim
    runs = []
    for num_tasks in (None, 1):
        m = _make(net, use_lstm, precision, num_tasks=num_tasks)
        actor = _make(net, use_lstm, precision, num_tasks=num_tasks)
        opt = optim.RMSprop(m, lr=0.00048, eps=0.01, alpha=0.99)
        flags = types.SimpleNamespace(popart_beta=0.0, **FLAGS)
        stats = [learner.learn(flags, m, actor, _batch(T, B, net, seed), _state(m, B), opt, None) for seed in (1, 2)]
        torch.cuda.synchronize()
        runs.append((m, actor, opt, stats))
    (m0, a0, o0, s0), (m1, a1, o1, s1) = runs
    assert torch.equal(m0.flat_params, m1.flat_params)
    assert torch.equal(a1.flat_params, m1.flat_params)
    assert all(torch.equal(x, y) for x, y in zip(o0.flat_state(), o1.flat_state()))
    for a, b in zip(s0, s1):
        for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
            assert a[k] == b[k], k
        assert b["popart_mu"] == [0.0] and b["popart_sigma"] == [1.0]
    assert float(m1.popart.mu) == 0.0 and float(m1.popart.nu) == 1.0


def _loss_inputs(T, B, K, seed, drop_col=None):
    """Shifted loss inputs, normalised values [T+1, B, K] and tasks, statistics with sigma in 1e-2 .. 1e3."""
    rs = np.random.RandomState(seed)
    d = dict(
        blogits=rs.randn(T, B, A).astype(np.float32), tlogits=rs.randn(T, B, A).astype(np.float32),
        actions=rs.randint(0, A, size=(T, B)).astype(np.int64), rewards=(rs.randn(T, B) * 30).astype(np.float32),
        done=rs.rand(T, B) < 0.05, n=rs.randn(T + 1, B, K).astype(np.float32))
    task = rs.randint(0, K, size=(T + 1, B)).astype(np.int64)
    task = np.repeat(task[:1], T + 1, axis=0)  # one task per column ...
    s = T // 2
    task[s:, 0] = (task[0, 0] + 1) % K         # ... except column 0, which switches task where an episode ends
    d["done"][s - 1, 0] = True
    if drop_col is not None:
        task[:, drop_col] = -1
    d["task"] = task
    mu = rs.randn(K) * 50.0
    sig = 10.0 ** np.linspace(-2, 3, K)
    d["mu"], d["nu"] = mu, sig * sig + mu * mu
    return d


def _gpu_loss(d, hparams_dev=None, reward_clipping="none"):
    from torchbeast_b200 import learner
    cu = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return learner.impala_loss_popart(cu(d["blogits"]), cu(d["tlogits"]), cu(d["actions"]), cu(d["rewards"]),
                                      cu(d["done"]), cu(d["n"]), cu(d["task"]), cu(d["mu"]), cu(d["nu"]),
                                      reward_clipping=reward_clipping, hparams_dev=hparams_dev)


def _oracle_loss(d, cols=None):
    cols = slice(None) if cols is None else cols
    t = lambda x, dt=None: torch.from_numpy(np.ascontiguousarray(x[:, cols]))
    n = t(d["n"]).double().requires_grad_(True)
    tl = t(d["tlogits"]).double().requires_grad_(True)
    hyper = type("H", (LT.Hyper,), dict(reward_clipping="none"))
    o = PO.popart_losses(t(d["blogits"]).double(), tl, t(d["actions"]), t(d["rewards"]), t(d["done"]), n, t(d["task"]),
                         torch.from_numpy(d["mu"]), torch.from_numpy(d["nu"]), hyper)
    gl, gn = torch.autograd.grad(o["total_loss"], [tl, n])
    return o, gl, gn


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("T,B", [(80, 32), (4, 64), (20, 7)])  # T-split scan, wide scan (T <= 4), ragged tile
def test_loss_and_update_match_fp64_oracle(T, B):
    from torchbeast_b200 import learner
    K = 4
    d = _loss_inputs(T, B, K, seed=T + B)
    loss, sums = _gpu_loss(d)
    o, gl, gn = _oracle_loss(d)
    got = loss.losses.cpu().double()
    for i, k in enumerate(("pg_loss", "baseline_loss", "entropy_loss")):
        np.testing.assert_allclose(float(got[i]), float(o[k]), rtol=1e-5, atol=1e-6, err_msg=k)
    vs = o["vs"].numpy()
    np.testing.assert_allclose(loss.vs.cpu().numpy(), vs, rtol=1e-5, atol=1e-5 * np.abs(vs).max())
    assert _rel(loss.grad_logits[:-1], gl) < 1e-4
    assert _rel(loss.grad_values[:-1], gn[:-1]) < 1e-4
    assert torch.count_nonzero(loss.grad_values[-1]) == 0
    # only the column of the row's task carries gradient
    onehot = torch.nn.functional.one_hot(torch.from_numpy(d["task"]), K).bool().cuda()
    assert torch.count_nonzero(loss.grad_values[~onehot]) == 0
    np.testing.assert_allclose(sums.cpu().numpy(), o["task_sums"].numpy(), rtol=1e-5, atol=1e-3)
    # the update on the kernel's sums against the oracle's update on the oracle's sums
    mu, nu = torch.from_numpy(d["mu"]).cuda(), torch.from_numpy(d["nu"]).cuda()
    W, b = torch.randn(K, 519, device="cuda"), torch.randn(K, device="cuda")
    mu2, nu2, _, _ = PO.popart_update(o["task_sums"], 0.1, mu.cpu(), nu.cpu(), W.cpu(), b.cpu())
    learner.popart_update(sums, torch.full((1,), 0.1, dtype=torch.float64, device="cuda"), mu, nu, W, b)
    np.testing.assert_allclose(mu.cpu().numpy(), mu2.numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(nu.cpu().numpy(), nu2.numpy(), rtol=1e-5)


@pytest.mark.parametrize("T,B", [(80, 32), (4, 64)])
def test_hparams_block_and_determinism(T, B):
    from torchbeast_b200 import learner
    d = _loss_inputs(T, B, 4, seed=7)
    flags = types.SimpleNamespace(**dict(FLAGS, reward_clipping="none"))
    block = torch.zeros(learner.HPARAMS.itemsize, dtype=torch.uint8, device="cuda")
    learner.publish_hparams(learner.pack_hparams(flags), block)
    a, sa = _gpu_loss(d)
    b, sb = _gpu_loss(d)
    c, sc = _gpu_loss(d, hparams_dev=block)
    for x, y in ((a, b), (a, c)):
        for f in x._fields:
            assert torch.equal(getattr(x, f), getattr(y, f)), f
    assert torch.equal(sa, sb) and torch.equal(sa, sc)


def test_out_of_range_task_column():
    T, B, K = 20, 6, 4
    d = _loss_inputs(T, B, K, seed=3, drop_col=2)
    loss, sums = _gpu_loss(d)
    assert torch.count_nonzero(loss.grad_values[:, 2]) == 0
    assert torch.count_nonzero(loss.grad_logits[:, 2]) == 0
    o, _, _ = _oracle_loss(d, cols=[0, 1, 3, 4, 5])
    got = loss.losses.cpu().double()
    for i, k in enumerate(("pg_loss", "baseline_loss", "entropy_loss")):
        np.testing.assert_allclose(float(got[i]), float(o[k]), rtol=1e-5, atol=1e-6, err_msg=k)
    np.testing.assert_allclose(sums.cpu().numpy(), o["task_sums"].numpy(), rtol=1e-5, atol=1e-3)


def test_update_alone_preserves_outputs():
    from torchbeast_b200 import learner
    rs = np.random.RandomState(11)
    K, F = 4, 519
    mu = torch.from_numpy(rs.randn(K) * 20).cuda()
    sig = torch.from_numpy(10.0 ** np.linspace(-2, 3, K)).cuda()
    nu = sig * sig + mu * mu
    W = (torch.randn(K, F, device="cuda") / 20).contiguous()
    b = torch.randn(K, device="cuda")
    sums = torch.tensor([[10.0, 3.0, 0.0, 7.0], [40.0, -600.0, 0.0, 1e3], [900.0, 1.5e5, 0.0, 2e6]],
                        dtype=torch.float64, device="cuda")  # task 2 absent
    x = torch.randn(64, F, dtype=torch.float64)
    out = lambda W, b, mu, nu: PO.sigma(mu.cpu(), nu.cpu()) * (x @ W.cpu().double().t() + b.cpu().double()) + mu.cpu()
    before = out(W, b, mu, nu)
    mu0, nu0, W0, b0 = mu.clone(), nu.clone(), W.clone(), b.clone()
    learner.popart_update(sums, torch.full((1,), 0.3, dtype=torch.float64, device="cuda"), mu, nu, W, b)
    after = out(W, b, mu, nu)
    np.testing.assert_allclose(after.numpy(), before.numpy(), rtol=1e-6, atol=1e-6 * float(before.abs().max()))
    mu2, nu2, _, _ = PO.popart_update(sums.cpu(), 0.3, mu0.cpu(), nu0.cpu(), W0.cpu(), b0.cpu())
    np.testing.assert_allclose(mu.cpu().numpy(), mu2.numpy(), rtol=1e-12)
    np.testing.assert_allclose(nu.cpu().numpy(), nu2.numpy(), rtol=1e-12)
    assert torch.equal(W[2], W0[2]) and torch.equal(b[2], b0[2]) and float(mu[2]) == float(mu0[2])


def test_graph_replay_matches_eager():
    from torchbeast_b200 import learner, optim
    T, B = 8, 4
    runs = []
    for graph in (False, True):
        m, actor = _make("atari", True, None, num_tasks=4), _make("atari", True, None, num_tasks=4)
        opt = optim.RMSprop(m, lr=0.00048, eps=0.01, alpha=0.99)
        flags = types.SimpleNamespace(cuda_graph=graph, **dict(FLAGS, reward_clipping="none"))
        out = []
        for k in range(5):
            flags.popart_beta = (0.3, 0.0, 0.05, 1e-3, 0.5)[k]
            batch = _batch(T, B, "atari", seed=20 + k)
            batch["reward"] = batch["reward"] * 40.0
            task = ((torch.arange(B, device="cuda") + k) % 4).expand(T + 1, B).clone()
            task[:, k % B] = -1                      # the task mix changes every step
            batch["task"] = task
            stats = learner.learn(flags, m, actor, batch, _state(m, B), opt, None)
            torch.cuda.synchronize()
            out.append((stats, m.flat_params.clone(), m.popart.mu.clone(), m.popart.nu.clone()))
        runs.append(out)
    for (se, pe, mue, nue), (sg, pg, mug, nug) in zip(*runs):
        for key in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss", "popart_mu", "popart_sigma"):
            assert se[key] == sg[key], key
        assert torch.equal(pe, pg) and torch.equal(mue, mug) and torch.equal(nue, nug)
    assert bool((runs[0][-1][2] != 0).any())  # the statistics moved


@pytest.mark.parametrize("B", [1, 48])
def test_acting_graph_matches_eager(B):
    from torchbeast_b200.acting import GraphedActor, bucket_size
    net = _make("atari", True, None, num_tasks=57)
    net.eval()
    step = LT.synthetic_batch(0, B, A, seed=5)
    real = {k: step[k].cuda() for k in ("frame", "reward", "done", "last_action")}
    hc = tuple(0.1 * torch.randn(2, B, 512 + A + 1, device="cuda") for _ in range(2))
    g_out, g_state = GraphedActor(net)(real, hc)
    Bk = bucket_size(B)
    pad = lambda t: torch.cat([t, torch.zeros_like(t[:, :1]).expand(-1, Bk - B, *t.shape[2:])], dim=1)
    with torch.no_grad():
        e_out, e_state = net({k: pad(v) for k, v in real.items()}, tuple(pad(s) for s in hc))
    assert tuple(g_out["baseline"].shape) == (1, B, 57)
    for k in ("policy_logits", "baseline", "action"):
        assert torch.equal(g_out[k], e_out[k][:, :B]), k
    assert all(torch.equal(g, e[:, :B]) for g, e in zip(g_state, e_state))


@pytest.mark.parametrize("precision", [None, "fp32"])
@pytest.mark.parametrize("net,use_lstm", [("atari", True), ("resnet", False)])
@pytest.mark.parametrize("K", [1, 4])
def test_learn_step_matches_oracle(net, use_lstm, precision, K):
    """A whole learn step with beta > 0, unclipped rewards, statistics away from identity and K value outputs, against
    the restatement: the optimizer step, then the statistics update and the head rescale, then the actor copy."""
    from torchbeast_b200 import learner, nets, optim
    T, B, beta = 4, 3, 0.1
    batch = LT.synthetic_batch(T, B, A, seed=9, with_last_action=(net == "atari"))
    batch["reward"] = batch["reward"] * 5.0
    task = torch.zeros(T + 1, B, dtype=torch.int64)
    if K > 1:
        task[:, 0], task[2:, 0], task[:, 1], task[:, 2] = 1, 3, 0, -1
        batch["done"][2, 0] = True  # column 0 switches task where an episode ends
    batch["task"] = task
    shapes = LT.atarinet_param_shapes(A, use_lstm) if net == "atari" else LT.resnet_param_shapes(A, use_lstm)
    F = shapes["baseline.weight"][1]
    shapes.update({"baseline.weight": (K, F), "baseline.bias": (K,)})
    p = LT.random_params(shapes, seed=12)
    mu = torch.tensor([0.5, -2.0, 3.0, 10.0][:K], dtype=torch.float64)
    sig = torch.tensor([0.5, 2.0, 5.0, 20.0][:K], dtype=torch.float64)
    nu = sig * sig + mu * mu
    state = ()
    if use_lstm:
        state = tuple(0.1 * torch.randn(2, B, 512 + A + 1, generator=torch.Generator().manual_seed(3)) for _ in range(2))
    hyper = type("H", (LT.Hyper,), dict(reward_clipping="none"))
    ref = PO.learner_step(p, batch, state, hyper=hyper, net=net, num_actions=A, mu=mu, nu=nu, beta=beta, task=task)

    model, actor = _make(net, use_lstm, precision, num_tasks=K), _make(net, use_lstm, precision, num_tasks=K)
    model.load_state_dict(dict(p, **{"popart.mu": mu, "popart.nu": nu}))
    opt = optim.RMSprop(model, lr=LT.Hyper.learning_rate, eps=LT.Hyper.epsilon, alpha=LT.Hyper.alpha)
    flags = types.SimpleNamespace(popart_beta=beta, **dict(FLAGS, reward_clipping="none"))
    stats = learner.learn(flags, model, actor, {k: v.cuda() for k, v in batch.items()},
                          tuple(s.cuda() for s in state), opt, None)
    torch.cuda.synchronize()
    tol = 2e-4
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(stats[k], float(ref[k]), rtol=tol, atol=tol, err_msg=k)
    np.testing.assert_allclose(model.popart.mu.cpu().numpy(), ref["mu"].numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(model.popart.nu.cpu().numpy(), ref["nu"].numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(stats["popart_mu"], ref["mu"].tolist(), rtol=1e-5, atol=1e-6)
    sd = model.state_dict()
    for n in ("baseline.weight", "baseline.bias", "policy.bias", "fc.bias"):
        np.testing.assert_allclose(sd[n].cpu().numpy(), ref["params"][n].numpy(), rtol=1e-3, atol=1e-5, err_msg=n)
    assert torch.equal(actor.flat_params, model.flat_params)
    assert torch.equal(actor.popart.mu, model.popart.mu) and torch.equal(actor.popart.nu, model.popart.nu)
    if K > 1:
        assert float(model.popart.mu[2]) == float(mu[2])  # task 2 is absent from the batch
