"""GPU: legal-action masks (torchbeast_b200.legal_actions).  The masking launch (tb_mask_logits_f32) against its NumPy
restatement, bit for bit; acting with a mask, eager and through GraphedActor, against the sampling oracle; an all-legal
mask giving the bits of the step without the leaf, eager and graphed; an always-illegal action getting no gradient;
learn_step under a random mask against the float64 oracle of tests/legal_actions_oracle.py on every loss path; an
illegal taken action poisoning the losses; replay storing and mixing the leaf; and the autograd forward's gradients."""
import gc
import types

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from oracle import sampling_np as SO
from tests import legal_actions_oracle as LO

pytestmark = pytest.mark.gpu

A = 6
FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


@pytest.fixture(autouse=True)
def _collect_graphs():
    yield
    gc.collect()
    torch.cuda.synchronize()


def _legal(shape, seed, p=0.6):
    """A random mask with at least one legal action per row, an all-legal row and (for rows > 1) an all-illegal one."""
    rs = np.random.RandomState(seed)
    legal = rs.rand(*shape) < p
    rows = legal.reshape(-1, shape[-1])
    rows[np.arange(rows.shape[0]), rs.randint(0, shape[-1], rows.shape[0])] = True
    rows[0] = True
    if rows.shape[0] > 1:
        rows[-1] = False
    return legal


def _legal_choice(legal, seed):
    """One action per row, legal where the row has a legal action."""
    rs = np.random.RandomState(seed)
    out = np.zeros(legal.shape[:-1], np.int64)
    for idx in np.ndindex(*legal.shape[:-1]):
        ok = np.flatnonzero(legal[idx])
        out[idx] = rs.choice(ok if ok.size else np.arange(legal.shape[-1]))
    return out


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(
        np.where(np.isnan(a), 0, a).view(np.int32), np.where(np.isnan(b), 0, b).view(np.int32))


# ---- the masking launch -----------------------------------------------------------------------------------------


@pytest.mark.parametrize("N,A_", [(1, 2), (81 * 32, 2), (81 * 32, 6), (601 * 128, 6), (81 * 32, 18), (601 * 128, 18),
                                  (77, 23), (81 * 32, 23), (5, 362), (81 * 32, 362)])
def test_kernel_matches_numpy_bit_for_bit(N, A_):
    from torchbeast_b200.legal_actions import MASKED_LOGIT, mask_logits
    rs = np.random.RandomState(N + A_)
    x = (3 * rs.randn(N, A_)).astype(np.float32)
    legal = _legal((N, A_), N * 7 + A_)
    legal[1::5] = True                                  # all-legal rows
    legal[2::7] = False                                 # rows with no legal action
    actions = _legal_choice(legal, 3)
    bad = rs.rand(N) < 0.05                             # illegal taken actions, and a few out of range
    for i in np.flatnonzero(bad):
        ill = np.flatnonzero(~legal[i])
        actions[i] = rs.choice(ill) if ill.size else A_ + 3
    actions[::11] = -1
    xd, ld, ad = torch.from_numpy(x).cuda(), torch.from_numpy(legal).cuda(), torch.from_numpy(actions).cuda()
    for l in (ld, ld.to(torch.uint8) * 7):               # bool, and uint8 with any nonzero value for legal
        out = mask_logits(xd, l)
        assert _bits_equal(out.cpu().numpy(), LO.mask_logits(x, legal)) and out.data_ptr() != xd.data_ptr()
        assert torch.equal(xd.cpu(), torch.from_numpy(x))              # out of place: the input is untouched
        got = mask_logits(xd, l, actions=ad).cpu().numpy()
        want = LO.mask_logits(x, legal, actions)
        assert _bits_equal(got, want)
        assert np.isnan(want).any(axis=-1).sum() > 0 or N < 20
        assert np.array_equal(got.min(-1) == np.float32(MASKED_LOGIT), (~legal & legal.any(-1, keepdims=True)).any(-1)
                              & ~np.isnan(want).any(-1))
        g = mask_logits(xd, l, fill=0.0).cpu().numpy()                 # the gradient's fill
        assert _bits_equal(g, LO.mask_logits(x, legal, fill=np.float32(0)))
        inplace = xd.clone()
        ret = mask_logits(inplace, l, actions=ad, out=inplace)
        assert ret.data_ptr() == inplace.data_ptr() and _bits_equal(inplace.cpu().numpy(), want)


def test_kernel_leaves_other_memory_and_repeats_bit_identically():
    from torchbeast_b200.legal_actions import mask_logits
    N, A_ = 1000, 18
    x = torch.randn(N + 2, A_, device="cuda")
    legal = torch.from_numpy(_legal((N, A_), 5)).cuda()
    out = torch.full((N + 2, A_), 7.0, device="cuda")
    mask_logits(x[1:-1], legal, out=out[1:-1])
    mask_logits(x[1:-1], legal, out=out[1:-1])
    assert torch.all(out[0] == 7.0) and torch.all(out[-1] == 7.0)
    assert _bits_equal(out[1:-1].cpu().numpy(), LO.mask_logits(x[1:-1].cpu().numpy(), legal.cpu().numpy()))


# ---- acting --------------------------------------------------------------------------------------------------------


def _acting_net(kind, seed):
    from torchbeast_b200 import monobeast, polybeast_learner
    if kind == "atari":
        model = monobeast.AtariNet((4, 84, 84), A, True)
        params = LT.random_params(LT.atarinet_param_shapes(A, True), seed=seed)
    else:
        model = polybeast_learner.Net(A, True)
        params = LT.random_params(LT.resnet_param_shapes(A, True), seed=seed)
    model.load_state_dict(params)
    return model


def _acting_inputs(model, B, seed):
    batch = LT.synthetic_batch(0, B, A, seed=seed, with_last_action=getattr(model, "needs_last_action", False))
    names = ("frame", "reward", "done", "last_action") if getattr(model, "needs_last_action", False) \
        else ("frame", "reward", "done")
    inputs = {k: batch[k].cuda() for k in names}
    legal = _legal((1, B, A), seed + 1, p=0.4)
    inputs["legal_actions"] = torch.from_numpy(legal).cuda()
    g = torch.Generator().manual_seed(seed)
    state = tuple((0.1 * torch.randn(s.shape, generator=g)).cuda() for s in model.initial_state(B))
    return inputs, state, legal


def _action_and_logits(kind, out):
    out = out[0]
    return (out["action"], out["policy_logits"]) if kind == "atari" else (out[0], out[1])


@pytest.mark.parametrize("kind", ["atari", "resnet"])
@pytest.mark.parametrize("B", [1, 48, 512])
def test_acting_samples_and_argmax_are_legal(kind, B):
    from torchbeast_b200.acting import GraphedActor
    from torchbeast_b200.sampling import ActionSampler
    model = _acting_net(kind, 11)
    model.train()
    inputs, state, legal = _acting_inputs(model, B, 100 + B)
    actor = GraphedActor(model)
    seed = 2024
    compared = 0
    for call in range(3):
        for graphed in (False, True):
            model.action_sampler = ActionSampler(seed, 10 * call)
            with torch.no_grad():
                out = actor(inputs, state) if graphed else model(inputs, state)
            action, logits = _action_and_logits(kind, out)
            a, x = action.cpu().numpy(), logits.cpu().numpy()
            assert _bits_equal(x, LO.mask_logits(x, legal))              # the forward's logits are masked
            assert np.all(np.take_along_axis(LO.keep(legal), a[..., None], -1))   # every sampled action is legal
            want, margin = SO.sample_actions(x, seed, 10 * call)
            ok = margin >= SO.margin_threshold(A)
            assert np.array_equal(a[ok], want[ok])
            compared += int(ok.sum())
    assert compared >= 0.9 * 6 * B
    # the graph and the eager forward agree on the masked logits; without the leaf the graph is another one
    captures = actor.captures
    plain = {k: v for k, v in inputs.items() if k != "legal_actions"}
    with torch.no_grad():
        actor(plain, state)
    assert actor.captures == captures + 1
    model.eval()
    for graphed in (False, True):
        with torch.no_grad():
            out = actor(inputs, state) if graphed else model(inputs, state)
        a = _action_and_logits(kind, out)[0].cpu().numpy()
        assert np.all(np.take_along_axis(LO.keep(legal), a[..., None], -1))


# ---- learning -----------------------------------------------------------------------------------------------------


def _net(kind, use_lstm, seed, precision=None, num_tasks=None):
    from torchbeast_b200 import monobeast, polybeast_learner
    if kind == "atari":
        m = monobeast.AtariNet((4, 84, 84), A, use_lstm, precision=precision, num_tasks=num_tasks)
    else:
        m = polybeast_learner.Net(A, use_lstm, precision=precision, num_tasks=num_tasks)
    m.reset_parameters_like_torch(seed=seed)
    return m


def _state(kind, use_lstm, B, seed):
    if not use_lstm:
        return ()
    layers, H = (2, 512 + A + 1) if kind == "atari" else (1, 256)
    g = torch.Generator().manual_seed(seed)
    return tuple((0.1 * torch.randn(layers, B, H, generator=g)).cuda() for _ in range(2))


def _learn_batch(kind, T, B, seed, legal=None):
    b = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=seed, done_prob=0.2,
                                                     with_last_action=kind == "atari").items()}
    if legal is not None:
        b["legal_actions"] = torch.from_numpy(legal).cuda()
        acts = _legal_choice(np.concatenate([legal[:1], legal[:-1]]), seed + 1)   # action[t+1] legal at frame t
        b["action"] = torch.from_numpy(acts).cuda()
        if kind == "atari":
            b["last_action"] = b["action"].clone()
    return b


def _opt(model):
    from torchbeast_b200 import optim
    return optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)


def _eager(kind, use_lstm, seed, batch, state, flags, precision=None, **kw):
    """learn_step on a fresh net; host copies of the losses, grad_logits, the flat parameters after the step, and the
    step's raw output."""
    from torchbeast_b200 import learner
    model = _net(kind, use_lstm, seed, precision)
    out = learner.learn_step(flags, model, None, batch, state, _opt(model), None, stats_sync=False, **kw)
    torch.cuda.synchronize()
    return dict(losses=out["losses"].cpu().numpy(), grad=out["vtrace"].grad_logits.cpu().numpy(),
                params=model.flat_params.cpu().numpy(), out=out, model=model)


def _graphed(kind, use_lstm, seed, batch, state, flags, precision=None, steps=1):
    from torchbeast_b200 import learner
    model = _net(kind, use_lstm, seed, precision)
    opt = _opt(model)
    f = types.SimpleNamespace(**vars(flags), cuda_graph=True)
    for _ in range(steps):
        learner.learn(f, model, None, batch, state, opt, None)
    torch.cuda.synchronize()
    (gl,) = model._tb_graphs.values()
    return dict(losses=gl.out["losses"].cpu().numpy(), grad=gl.out["vtrace"].grad_logits.cpu().numpy(),
                params=model.flat_params.cpu().numpy())


@pytest.mark.parametrize("kind", ["atari", "resnet"])
@pytest.mark.parametrize("graphed", [False, True])
def test_all_legal_mask_gives_the_bits_of_the_step_without_it(kind, graphed):
    T, B = 6, 4
    flags = types.SimpleNamespace(**FLAGS)
    run = _graphed if graphed else _eager
    batch = _learn_batch(kind, T, B, 5)
    state = _state(kind, True, B, 6)
    off = run(kind, True, 3, batch, state, flags)
    on = run(kind, True, 3, dict(batch, legal_actions=torch.ones(T + 1, B, A, dtype=torch.bool, device="cuda")), state,
             flags)
    for k in ("losses", "grad", "params"):
        assert _bits_equal(on[k], off[k]), k


def test_an_always_illegal_action_gets_no_policy_gradient():
    from torchbeast_b200.kickstart import Teacher
    T, B = 8, 5
    legal = _legal((T + 1, B, A), 9)
    legal[..., 2] = False                 # action 2 is never legal ...
    legal[~legal.any(-1), 0] = True       # ... and every row has a legal action, so every row masks it
    batch = _learn_batch("atari", T, B, 10, legal)
    flags = types.SimpleNamespace(**dict(FLAGS, entropy_cost=0.01), upgo_cost=0.5, kickstart_cost=0.8)
    from torchbeast_b200 import learner
    model = _net("atari", True, 3)
    model.teacher = Teacher(_net("atari", False, 4))
    learner.learn_step(flags, model, None, batch, _state("atari", True, B, 1), _opt(model), None, stats_sync=False)
    torch.cuda.synchronize()
    gw, gb = model.policy.weight.grad, model.policy.bias.grad
    assert torch.all(gw[2] == 0) and gb[2] == 0
    assert torch.count_nonzero(gw[[0, 1, 3, 4, 5]]) > 0 and torch.count_nonzero(gb) == A - 1


def _oracle_inputs(kind, use_lstm, T, B, seed, num_tasks=None):
    """A masked batch, its state, and the raw (unmasked) forward of a fresh fp32 net on it: logits and baseline."""
    legal = _legal((T + 1, B, A), seed)
    batch = _learn_batch(kind, T, B, seed, legal)
    state = _state(kind, use_lstm, B, seed + 1)
    net = _net(kind, use_lstm, 3, "fp32", num_tasks)
    raw = net.learner_forward({k: v for k, v in batch.items() if k != "legal_actions"}, state)
    logits, baseline = raw.policy_logits.cpu().numpy(), raw.baseline.cpu().numpy()
    return legal, batch, state, logits, baseline.reshape(T + 1, B)


def _oracle_of(batch, legal, logits, baseline, beta=None, mask=None, weights=None):
    h = {k: v.cpu().numpy() for k, v in batch.items()}
    rewards = np.clip(h["reward"][1:].astype(np.float64), -1, 1)
    discounts = (~h["done"][1:]).astype(np.float64) * FLAGS["discounting"]
    return LO.loss(h["policy_logits"][1:], logits[:-1], h["action"][1:], rewards, discounts, baseline[:-1], baseline[-1],
                   legal[:-1], beta=beta, mask=mask, weights=weights), rewards, discounts


@pytest.mark.parametrize("path", ["plain", "trust_region", "upgo", "kickstart", "popart", "weights"])
def test_learn_step_under_a_random_mask_matches_the_oracle(path):
    from torchbeast_b200 import learner, replay
    from torchbeast_b200.kickstart import Teacher
    T, B = 7, 5
    legal, batch, state, logits, baseline = _oracle_inputs("atari", False, T, B, 31,
                                                           num_tasks=1 if path == "popart" else None)
    kw, extra = {}, {}
    w = None
    if path == "trust_region":   # beta between the rows' KLs, so that both sides of the rule are covered
        beta = float(np.median(_oracle_of(batch, legal, logits, baseline)[0]["kl"]))
        extra["trust_region_kl"] = beta
    if path == "upgo":
        extra["upgo_cost"] = 0.7
    if path == "kickstart":
        extra["kickstart_cost"] = 0.9
    if path == "weights":
        w = np.random.RandomState(4).rand(B).astype(np.float32)
        kw["draw"] = replay.Draw(None, torch.from_numpy(w).cuda(), None)
    flags = types.SimpleNamespace(**FLAGS, **extra)
    model = _net("atari", False, 3, "fp32", num_tasks=1 if path == "popart" else None)
    teacher_logits = None
    if path == "kickstart":
        tnet = _net("atari", False, 8, "fp32")
        model.teacher = Teacher(tnet)
        teacher_logits = tnet.learner_forward({k: v for k, v in batch.items() if k != "legal_actions"}).policy_logits
        teacher_logits = teacher_logits.cpu().numpy()
    out = learner.learn_step(flags, model, None, batch, state, _opt(model), None, stats_sync=False, **kw)
    torch.cuda.synchronize()
    losses, grad = out["losses"].cpu().numpy().astype(np.float64), out["vtrace"].grad_logits.cpu().numpy()
    mask = None
    if path == "trust_region":
        kl = out["trust"].kl.cpu().numpy()
        mask = kl <= beta
        assert 0 < mask.sum() < T * B
    o, rewards, discounts = _oracle_of(batch, legal, logits, baseline, mask=mask, weights=w)
    want_losses, want_grad = o["losses"].copy(), o["grad_logits"].copy()
    if path == "trust_region":
        np.testing.assert_allclose(kl, o["kl"], rtol=1e-4, atol=1e-5)
    if path == "upgo":
        u = LO.upgo(logits[:-1], batch["action"][1:].cpu().numpy(), rewards, discounts, baseline[:-1], baseline[-1],
                    o["log_rhos"], legal[:-1], 0.7)
        np.testing.assert_allclose(out["upgo"].loss.cpu().numpy()[0], u["loss"], rtol=1e-4, atol=1e-5)
        want_losses[3] += u["loss"]
        want_grad += u["grad_logits"]
    if path == "kickstart":
        k = LO.kickstart(teacher_logits[:-1], logits[:-1], legal[:-1], 0.9)
        np.testing.assert_allclose(out["kickstart"].loss.cpu().numpy()[0], k["loss"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(out["kickstart"].kl_sum.cpu().numpy()[0], k["kl_sum"], rtol=1e-4, atol=1e-5)
        want_losses[3] += k["loss"]
        want_grad += k["grad_logits"]
    scale = np.abs(want_losses).max()
    np.testing.assert_allclose(losses, want_losses, rtol=1e-4, atol=1e-5 * scale)
    np.testing.assert_allclose(grad[:T], want_grad, rtol=1e-4, atol=1e-5)
    assert np.all(grad[:T][~LO.keep(legal[:-1])] == 0)            # +-0 at every illegal entry
    assert np.all(grad[T] == 0)


def test_behaviour_logits_raw_minus_inf_or_sentinel_give_the_same_bits():
    from torchbeast_b200.legal_actions import MASKED_LOGIT
    T, B = 7, 5
    legal, batch, state, _, _ = _oracle_inputs("atari", True, T, B, 41)
    flags = types.SimpleNamespace(**FLAGS, trust_region_kl=0.5, upgo_cost=0.3)
    runs = []
    illegal = torch.zeros(T + 1, B, A, dtype=torch.bool, device="cuda")
    illegal[1:] = ~torch.from_numpy(LO.keep(legal[:-1])).cuda()
    for fill in (None, float("-inf"), MASKED_LOGIT):
        b = dict(batch)
        if fill is not None:
            b["policy_logits"] = batch["policy_logits"].masked_fill(illegal, fill)
        runs.append(_eager("atari", True, 3, b, state, flags, "bf16x3"))
    for r in runs[1:]:
        for k in ("losses", "grad", "params"):
            assert _bits_equal(r[k], runs[0][k]), k
    assert np.all(np.isfinite(runs[0]["losses"]))


def test_an_illegal_taken_action_makes_the_losses_nan():
    T, B = 6, 4
    legal = _legal((T + 1, B, A), 51)
    t, b = 3, 2                                    # action row t+1 is checked against legal row t
    legal[t, b, :2] = (True, False)
    batch = _learn_batch("atari", T, B, 52, legal)
    flags = types.SimpleNamespace(**FLAGS)
    ok = _eager("atari", False, 3, batch, (), flags)
    assert np.all(np.isfinite(ok["losses"]))
    acts = batch["action"].clone()
    acts[t + 1, b] = 1
    r = _eager("atari", False, 3, dict(batch, action=acts), (), flags)
    assert np.isnan(r["losses"][0]) and np.isnan(r["losses"][3])


def test_replay_stores_and_mixes_the_leaf_and_graphed_equals_eager():
    from torchbeast_b200 import learner
    from torchbeast_b200.replay import ReplayBuffer
    T, Bf, R, cap = 5, 3, 2, 8
    flags = types.SimpleNamespace(**FLAGS, upgo_cost=0.2)
    batches = [_learn_batch("atari", T, Bf, 60 + i, _legal((T + 1, Bf, A), 70 + i, p=0.3 + 0.1 * i)) for i in range(6)]
    state = _state("atari", True, Bf, 7)
    # the mix: every replayed column carries the mask stored with it
    shadow = ReplayBuffer(cap, R, seed=5, min_size=2, stream_id=0)
    seen, mixed_calls = [], 0
    for b in batches:
        mixed, _, fresh = shadow.mix(b, state)
        seen += [(b["reward"][:, j], b["legal_actions"][:, j]) for j in range(Bf)]
        if fresh is not None:
            mixed_calls += 1
            for j in range(Bf, Bf + R):
                match = [lg for rw, lg in seen if torch.equal(rw, mixed["reward"][:, j])]
                assert match and torch.equal(mixed["legal_actions"][:, j], match[0])
    assert mixed_calls >= 3
    # learning with a buffer, eager and graphed, stays bit-identical across steps whose masks change
    runs = []
    for graphed in (False, True):
        model = _net("atari", True, 3)
        model.replay = ReplayBuffer(cap, R, seed=5, min_size=2, stream_id=0)
        opt = _opt(model)
        f = types.SimpleNamespace(**vars(flags), cuda_graph=graphed)
        stats = [learner.learn(f, model, None, b, state, opt, None) for b in batches]
        runs.append((stats, model.flat_params.cpu().numpy()))
    for s0, s1 in zip(runs[0][0], runs[1][0]):
        for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss", "upgo_loss"):
            assert np.float32(s0[k]).view(np.int32) == np.float32(s1[k]).view(np.int32), k
    assert _bits_equal(runs[0][1], runs[1][1])
    # a replayed column's loss uses its stored mask: the same mixed batch with all-legal replayed columns differs
    buf = ReplayBuffer(cap, R, seed=5, min_size=2, stream_id=0)
    for b in batches[:-1]:
        buf.mix(b, state)
    mixed, mstate, _ = buf.mix(batches[-1], state)
    assert mixed["reward"].shape[1] == Bf + R
    relaxed = mixed["legal_actions"].clone()
    relaxed[:, Bf:] = True
    assert not torch.equal(relaxed, mixed["legal_actions"])
    a = _eager("atari", True, 3, mixed, mstate, flags)
    b = _eager("atari", True, 3, dict(mixed, legal_actions=relaxed), mstate, flags)
    assert not _bits_equal(a["losses"], b["losses"])


@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_autograd_forward_gradients_match_float64_masked_fill(kind):
    T, B = 3, 4
    model = _net(kind, True, 3, "fp32")
    model.train()
    legal = _legal((T, B, A), 80)
    b = _learn_batch(kind, T - 1, B, 81)
    inputs = {k: v for k, v in b.items() if k in ("frame", "reward", "done", "last_action")}
    inputs["legal_actions"] = torch.from_numpy(legal).cuda()
    state = _state(kind, True, B, 82)
    rs = np.random.RandomState(83)
    c, cb = rs.randn(T, B, A), rs.randn(T, B)
    out, _ = model(inputs, state)
    logits, baseline = (out["policy_logits"], out["baseline"]) if kind == "atari" else (out[1], out[2])
    assert logits.requires_grad
    loss = (torch.softmax(logits, -1) * torch.from_numpy(c).float().cuda()).sum() + (
        baseline * torch.from_numpy(cb).float().cuda()).sum()
    loss.backward()
    p64 = {k: v.detach().double().cpu().requires_grad_(True) for k, v in model.state_dict().items()}
    hb = {k: v.cpu() for k, v in inputs.items()}
    s64 = tuple(s.double().cpu() for s in state)
    if kind == "atari":
        ref_logits, ref_base = LT.atarinet_forward(p64, hb["frame"], hb["reward"], hb["done"], hb["last_action"], s64,
                                                   A)[:2]
    else:
        ref_logits, ref_base = LT.resnet_forward(p64, hb["frame"], hb["reward"], hb["done"], s64, A)[:2]
    keep = torch.from_numpy(LO.keep(legal))
    ref = (torch.softmax(ref_logits.masked_fill(~keep, float("-inf")), -1) * torch.from_numpy(c)).sum() + (
        ref_base.reshape(T, B) * torch.from_numpy(cb)).sum()
    names = list(p64)
    grads = torch.autograd.grad(ref, [p64[n] for n in names], allow_unused=True)
    got_all = dict(model.named_parameters())
    for n, g in zip(names, grads):
        want = np.zeros(p64[n].shape) if g is None else g.numpy()
        got = got_all[n].grad.cpu().numpy()
        tol = 1e-4 * max(np.abs(want).max(), 1e-6)
        np.testing.assert_allclose(got, want, rtol=1e-3, atol=tol, err_msg=n)
    x = logits.detach().cpu().numpy()
    assert _bits_equal(x, LO.mask_logits(x, legal))
