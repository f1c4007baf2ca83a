"""GPU: the fused Adam / AdamW / centered and weight-decayed RMSprop steps against torch's optimizers in float64, the
device step counter, graphed = eager bit for bit through monobeast.learn, checkpoint resume, and the default RMSprop
configuration still launching its own kernel."""
import gc
import types

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)
A = 6


@pytest.fixture(autouse=True)
def _collect_graphs():
    """Models and the GraphedLearners stored on them reference each other: collect them between tests, so that no
    collection runs inside a later test's stream capture."""
    yield
    gc.collect()
    torch.cuda.synchronize()


def _net(seed=1):
    from torchbeast_b200 import monobeast
    m = monobeast.AtariNet((4, 84, 84), A, True)
    m.reset_parameters_like_torch(seed=seed)
    return m


# (name, ours, torch reference, {state key: decay of its recurrence}); the reference runs in float64 on the CPU
CONFIGS = [
    ("adam", lambda m, o: o.Adam(m, lr=1e-3), lambda ps: torch.optim.Adam(ps, lr=1e-3, foreach=False),
     {"exp_avg": 0.9, "exp_avg_sq": 0.999}),
    # eps 1e-4: see the parity test's docstring
    ("adam_l2", lambda m, o: o.Adam(m, lr=1e-3, eps=1e-4, weight_decay=0.05),
     lambda ps: torch.optim.Adam(ps, lr=1e-3, eps=1e-4, weight_decay=0.05, foreach=False),
     {"exp_avg": 0.9, "exp_avg_sq": 0.999}),
    ("adamw", lambda m, o: o.AdamW(m, lr=1e-3, betas=(0.8, 0.99), weight_decay=0.05),
     lambda ps: torch.optim.AdamW(ps, lr=1e-3, betas=(0.8, 0.99), weight_decay=0.05, foreach=False),
     {"exp_avg": 0.8, "exp_avg_sq": 0.99}),
    ("rmsprop_centered", lambda m, o: o.RMSprop(m, lr=4.8e-4, eps=1e-4, centered=True),
     lambda ps: torch.optim.RMSprop(ps, lr=4.8e-4, eps=1e-4, centered=True, foreach=False),
     {"square_avg": 0.99, "grad_avg": 0.99}),
    ("rmsprop_wd", lambda m, o: o.RMSprop(m, lr=4.8e-4, eps=1e-4, weight_decay=0.05),
     lambda ps: torch.optim.RMSprop(ps, lr=4.8e-4, eps=1e-4, weight_decay=0.05, foreach=False), {"square_avg": 0.99}),
    ("rmsprop_centered_momentum", lambda m, o: o.RMSprop(m, lr=4.8e-4, eps=1e-4, centered=True, momentum=0.9),
     lambda ps: torch.optim.RMSprop(ps, lr=4.8e-4, eps=1e-4, centered=True, momentum=0.9, foreach=False),
     {"square_avg": 0.99, "grad_avg": 0.99, "momentum_buffer": 0.9}),
]


@pytest.mark.parametrize("name,make_ours,make_ref,decays", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_parity_with_torch_float64(name, make_ours, make_ref, decays):
    """40 steps on the AtariNet+LSTM flat buffer (6.0 M parameters) with seeded random gradients whose norms are drawn
    from [20, 60], so the clip at 40 is active on some steps and not on others; LambdaLR decays the lr.  The reference
    is the torch optimizer in float64, fed our clip coefficient (recomputed in float32 from the norm the kernel
    reports, exactly as the kernel computes it).

    Tolerance, with u = 2^-24 the unit roundoff of float32 and N = 40 steps:
    * A state buffer follows x_k = d x_{k-1} + t_k (an EMA, or the momentum buffer).  Each float32 step rounds the
      product, the term and the sum, and the term t_k (from the clipped gradient, squared, or divided by avg) carries a
      few roundings more: the step adds at most c u (|x_{k-1}| + |t_k|) with c <= 8, and old errors are multiplied by
      d <= 1.  So |err(x_N)| <= 8 N u S, S = max_k (|x_{k-1}| + |t_k|) per element, read off the reference.  The
      momentum buffer's term divides by avg, which carries the square/gradient averages' own error (<= 8 N u
      relative): its bound is (8 N + 8) N u S.
    * The parameter: each step rounds p (<= 2 u |p|) and subtracts an update whose relative error is bounded by the
      state buffers' (<= 8 k u at step k) plus 8 roundings, i.e. <= (8 k + 8) u U_k with U_k the largest |update|
      of step k over all elements (the global maximum also covers elements where m cancels).  Summed:
      |err(p_N)| <= u (2 N max_k |p_k| + sum_k (8 k + 8) U_k).
    The bound needs the update to be well conditioned in its input.  With L2 weight decay the input g + wd p can
    cancel, leaving an absolute error u (|g| + |wd p|) on a tiny g'; Adam's update g'/(|g'| + eps) at step 1 then moves
    by that error over eps.  At eps = 1e-8 that is up to ~1e-3 of lr on a few of the 6.0 M elements, in torch's own
    float32 Adam as here.  The L2 case runs at eps = 1e-4, where that error is at most u |g| / eps ~ 1e-5 of lr per
    step, inside the bound above."""
    from torchbeast_b200 import optim
    N, u = 40, 2.0 ** -24
    model = _net()
    P = model.flat_params.numel()
    assert P > 5_900_000
    ref_p = torch.nn.Parameter(model.flat_params.detach().cpu().double())
    ours, ref = make_ours(model, optim), make_ref([ref_p])
    lam = lambda k: 1.0 - k / (2.0 * N)  # noqa: E731
    sched_ours = torch.optim.lr_scheduler.LambdaLR(ours, lam)
    sched_ref = torch.optim.lr_scheduler.LambdaLR(ref, lam)
    gen = torch.Generator(device="cuda").manual_seed(11)
    targets = 20.0 + 40.0 * torch.rand(N, generator=torch.Generator().manual_seed(12), dtype=torch.float64)
    p_max = ref_p.detach().abs().clone()
    update_term = 0.0
    S = {k: torch.zeros(P, dtype=torch.float64) for k in decays}
    clipped = 0
    for k in range(N):
        g = torch.randn(P, device="cuda", generator=gen)
        g *= float(targets[k]) / float(g.norm())
        model.flat_grad.copy_(g)
        ours.step(max_grad_norm=40.0)
        norm = np.float32(ours.grad_norm.item())
        coef = min(np.float32(40.0) / (norm + np.float32(1e-6)), np.float32(1.0))
        clipped += bool(coef < 1)
        prev_p = ref_p.detach().clone()
        prev = {key: ref.state[ref_p][key].clone() if ref.state[ref_p] else torch.zeros(P, dtype=torch.float64)
                for key in decays}
        ref_p.grad = g.cpu().double() * float(coef)
        ref.step()
        for key, d in decays.items():
            x = ref.state[ref_p][key]
            S[key] = torch.maximum(S[key], prev[key].abs() + (x - d * prev[key]).abs())
        update_term += (8 * (k + 1) + 8) * float((ref_p.detach() - prev_p).abs().max())
        p_max = torch.maximum(p_max, ref_p.detach().abs())
        sched_ours.step()
        sched_ref.step()
    assert 0 < clipped < N, clipped

    def check(what, got, want, tol):
        err = (got.detach().cpu().double() - want.detach()).abs()
        ratio = float((err / tol.clamp_min(1e-30)).max())
        print("%s %s: max |err| / tol = %.3g" % (name, what, ratio))
        assert ratio <= 1.0, (what, ratio)

    check("params", model.flat_params, ref_p, u * (2 * N * p_max + update_term))
    for key in decays:
        c = (8 * N + 8) * N if key == "momentum_buffer" else 8 * N
        check(key, getattr(ours, key), ref.state[ref_p][key], c * u * S[key])
    if hasattr(ours, "step_device"):
        assert int(ours.step_device) == N


def _batches(T, B, n, seed):
    return [{k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=seed + i).items()} for i in range(n)]


def _run(make_opt, batches, graph, model=None, opt=None, params_seed=3, lr_decay=True):
    """len(batches) monobeast.learn steps (T, B from the batches), with a LambdaLR when lr_decay; returns
    (model, optimizer)."""
    from torchbeast_b200 import monobeast, optim
    T, B = batches[0]["reward"].shape[0] - 1, batches[0]["reward"].shape[1]
    if model is None:
        model = _net(params_seed)
        opt = make_opt(model, optim)
    actor = _net(params_seed)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda k: 1.0 - k / 100.0) if lr_decay else None
    flags = types.SimpleNamespace(unroll_length=T, batch_size=B, cuda_graph=graph, **FLAGS)
    state = tuple(torch.zeros(2, B, 512 + A + 1, device="cuda") for _ in range(2))
    for b in batches:
        monobeast.learn(flags, actor, model, b, state, opt, sched)
    torch.cuda.synchronize()
    assert torch.equal(actor.flat_params, model.flat_params)
    return model, opt


OPTS = [
    ("adam", lambda m, o: o.Adam(m, lr=3e-4, weight_decay=0.01)),
    ("adamw", lambda m, o: o.AdamW(m, lr=3e-4)),
    ("rmsprop_centered_momentum", lambda m, o: o.RMSprop(m, lr=4.8e-4, eps=0.01, centered=True, momentum=0.5,
                                                         weight_decay=1e-4)),
]


@pytest.mark.parametrize("make_opt", [c[1] for c in OPTS], ids=[c[0] for c in OPTS])
def test_graphed_equals_eager(make_opt):
    """The graph replays the eager launch sequence, lr read from the device scalar: weights, state buffers and the
    device step are bit-identical, and the capture's warm-up steps leave no trace."""
    batches = _batches(8, 4, 4, seed=20)
    m_e, o_e = _run(make_opt, batches, graph=False)
    m_g, o_g = _run(make_opt, batches, graph=True)
    assert torch.equal(m_e.flat_params, m_g.flat_params)
    for a, b in zip(o_e.flat_state(), o_g.flat_state()):
        assert torch.equal(a, b)
    assert o_e.param_groups[0]["lr"] == o_g.param_groups[0]["lr"]
    if hasattr(o_g, "step_device"):
        assert int(o_g.step_device) == len(batches)


def test_device_step_counts_eager_steps_and_graph_replays():
    from torchbeast_b200 import optim
    make = lambda m, o: o.Adam(m, lr=3e-4)  # noqa: E731
    for graph in (False, True):
        for k in (1, 3):
            model, opt = _run(make, _batches(4, 2, k, seed=40), graph=graph)
            assert isinstance(opt, optim.Adam)
            assert all(int(opt.state[p]["step"]) == k for p, _, _, _ in model._views), (graph, k)
            assert all(float(s["step"]) == k for s in opt.state_dict()["state"].values()), (graph, k)


@pytest.mark.parametrize("graph", [False, True])
def test_resume_from_checkpoint_is_bit_identical(tmp_path, graph):
    """4 uninterrupted steps vs 2 steps, torch.save of model + optimizer, load into a fresh model and optimizer, 2 more.
    The resumed Adam takes its bias corrections from the loaded step (a graph captured after the load included)."""
    make = lambda m, o: o.AdamW(m, lr=3e-4, weight_decay=0.02)  # noqa: E731
    batches = _batches(8, 4, 4, seed=60)
    m_full, o_full = _run(make, batches, graph, lr_decay=False)
    m_half, o_half = _run(make, batches[:2], graph, lr_decay=False)
    f = tmp_path / "model.tar"
    torch.save({"model_state_dict": m_half.state_dict(), "optimizer_state_dict": o_half.state_dict()}, f)
    from torchbeast_b200 import optim
    ck = torch.load(f, weights_only=True)
    m_new = _net(seed=99)
    m_new.load_state_dict(ck["model_state_dict"])
    o_new = optim.AdamW(m_new, lr=1.0)
    o_new.load_state_dict(ck["optimizer_state_dict"])
    assert int(o_new.step_device) == 2 and o_new.param_groups[0]["lr"] == 3e-4
    m_new, o_new = _run(make, batches[2:], graph, model=m_new, opt=o_new, lr_decay=False)
    assert int(o_new.step_device) == 4
    assert torch.equal(m_new.flat_params, m_full.flat_params)
    for a, b in zip(o_new.flat_state(), o_full.flat_state()):
        assert torch.equal(a, b)


def test_launches_per_configuration():
    """The reference's RMSprop (centered=False, weight_decay=0) still runs clip_rmsprop_kernel; the other options run
    their own kernels.  Launch counts include tb_grad_sumsq_f32."""
    from torchbeast_b200 import _lib, optim
    lib = _lib.lib()
    cases = [(lambda m: optim.RMSprop(m, lr=4.8e-4, eps=0.01, alpha=0.99), "clip_rmsprop", 2),
             (lambda m: optim.RMSprop(m, lr=4.8e-4, eps=0.01, momentum=0.9), "clip_rmsprop", 2),
             (lambda m: optim.RMSprop(m, lr=4.8e-4, centered=True), "clip_rmsprop_ex", 2),
             (lambda m: optim.RMSprop(m, lr=4.8e-4, weight_decay=1e-4), "clip_rmsprop_ex", 2),
             (lambda m: optim.Adam(m), "clip_adam", 3),
             (lambda m: optim.AdamW(m), "clip_adam", 3)]
    model = _net()
    model.flat_grad.normal_()
    for make, record, launches in cases:
        opt = make(model)
        torch.cuda.synchronize()
        before = lib.tb_launch_count()
        lib.tb_profile_enable(1)
        opt.step(max_grad_norm=40.0)
        names = [n for n, _ in _lib.profile_collect()]
        lib.tb_profile_enable(0)
        assert lib.tb_launch_count() - before == launches, record
        assert names == ["grad_sumsq", record], names
