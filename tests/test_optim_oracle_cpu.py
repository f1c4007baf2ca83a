"""CPU: the float64 restatement of the fused optimizer step (tests/optim_oracle.py) against torch's clip_grad_norm_ and
torch.optim.RMSprop / Adam / AdamW in float64, for every option the kernels take, over chained steps that start from a
random state.  The GPU kernel tests trust this restatement, so it must agree with torch to a few float64 roundings."""
import itertools

import numpy as np
import pytest
import torch

from tests import optim_oracle as O

STEPS = 4
N = 1031
# per step: the clip threshold (None: no clipping) and the gradient's norm, so the clip is off, inactive and active
CLIPS = [(None, 60.0), (40.0, 20.0), (40.0, 60.0), (40.0, 160.0)]
RTOL = 1e-15


def _close(name, got, want, scale):
    """|got - want| <= 1e-15 (|want| + scale), scale the oracle's magnitude of the value: about four float64 roundings
    of the terms it is made of, where torch's lerp and addcmul fuse a multiply-add that NumPy rounds twice"""
    err = np.abs(got - want.numpy())
    ratio = float((err / (RTOL * (np.abs(want.numpy()) + scale) + 1e-300)).max())
    assert ratio <= 1.0, (name, ratio)


def _run(make_torch, oracle_step, t0, state0, seed):
    """STEPS torch steps from state0 at step t0; before each, the restatement takes torch's current state, and after
    it the two must agree"""
    rs = np.random.RandomState(seed)
    p = torch.nn.Parameter(torch.from_numpy(rs.randn(N) * 0.1))
    opt = make_torch([p])
    opt.state[p].update({k: torch.from_numpy(v.copy()) for k, v in state0.items()}, step=torch.tensor(float(t0)))
    for k, (max_norm, target) in enumerate(CLIPS):
        g = rs.randn(N)
        g *= target / np.linalg.norm(g)
        p.grad = torch.from_numpy(g.copy())
        coef = 1.0
        if max_norm is not None:
            total = torch.nn.utils.clip_grad_norm_([p], max_norm)
            coef = float(torch.clamp(max_norm / (total + 1e-6), max=1.0))  # the coefficient torch just applied
            assert (coef < 1.0) == (target > max_norm)
        clipped = p.grad.numpy().copy()
        before = {key: opt.state[p][key].numpy().copy() for key in state0}
        p_before = p.detach().numpy().copy()
        opt.step()
        new, mag = oracle_step(p_before, g, before, coef, t0 + k + 1)
        assert np.array_equal(new["g"], clipped)
        for key in state0:
            _close(key, new[key], opt.state[p][key], mag[key])
        _close("p", new["p"], p.detach(), mag["update"])
    assert float(opt.state[p]["step"]) == t0 + STEPS


RMSPROP = list(itertools.product([False, True], [0.0, 0.9], [0.0, 0.05]))


@pytest.mark.parametrize("centered,momentum,wd", RMSPROP,
                         ids=["centered%d_mom%g_wd%g" % c for c in RMSPROP])
def test_rmsprop_matches_torch(centered, momentum, wd):
    lr, alpha, eps = 4.8e-3, 0.99, 1e-4
    rs = np.random.RandomState(1)
    state0 = {"square_avg": rs.rand(N) * 0.1}
    if momentum:
        state0["momentum_buffer"] = rs.randn(N) * 0.1
    if centered:
        state0["grad_avg"] = rs.randn(N) * 0.01

    def make(ps):
        return torch.optim.RMSprop(ps, lr=lr, alpha=alpha, eps=eps, weight_decay=wd, momentum=momentum,
                                   centered=centered, foreach=False)

    def step(p, g, s, coef, t):
        return O.rmsprop_step(p, g, s["square_avg"], s.get("grad_avg"), s.get("momentum_buffer"), coef, lr, alpha,
                              eps, wd, momentum)

    _run(make, step, 3, state0, seed=2)


ADAM = [(d, wd, b, t0) for d in (False, True) for wd in (0.0, 0.05) for b in ((0.9, 0.999), (0.0, 0.999), (0.9, 0.0))
        for t0 in (0, 9, 10 ** 6)]


@pytest.mark.parametrize("decoupled,wd,betas,t0", ADAM,
                         ids=["%s_wd%g_b%g,%g_t%d" % ("adamw" if d else "adam", wd, b[0], b[1], t)
                              for d, wd, b, t in ADAM])
def test_adam_matches_torch(decoupled, wd, betas, t0):
    lr, eps = 1e-2, 1e-6
    rs = np.random.RandomState(3)
    state0 = {"exp_avg": rs.randn(N) * 0.1 * (t0 > 0), "exp_avg_sq": rs.rand(N) * 0.1 * (t0 > 0)}

    def make(ps):
        cls = torch.optim.AdamW if decoupled else torch.optim.Adam
        return cls(ps, lr=lr, betas=betas, eps=eps, weight_decay=wd, foreach=False)

    def step(p, g, s, coef, t):
        return O.adam_step(p, g, s["exp_avg"], s["exp_avg_sq"], coef, lr, betas[0], betas[1], eps, wd, decoupled, t)

    _run(make, step, t0, state0, seed=4)


def test_clip_coef_is_torchs_formula():
    """float32, within two roundings of torch's float64 coefficient (the norm + 1e-6 rounds in float32: at norm = 40
    the coefficient is exactly 1); exactly 1 below the threshold; 1 without a threshold"""
    rs = np.random.RandomState(5)
    for norm in np.concatenate([rs.rand(200) * 100.0, [0.0, 39.99996, 40.0, 40.00001, 1e30]]).astype(np.float32):
        c = O.clip_coef(norm, 40.0)
        assert c.dtype == np.float32
        want = float(torch.clamp(40.0 / (torch.tensor(float(norm), dtype=torch.float64) + 1e-6), max=1.0))
        assert abs(float(c) - want) <= 2.0 ** -23 * want, norm
        assert c <= 1.0 and (c == 1.0 or norm > 40.0)
        assert O.clip_coef(norm, -1.0) == 1.0


def test_clip_coef_propagates_nan_as_torch_does():
    """one NaN gradient element makes torch's whole clipped gradient NaN; one infinite element zeroes the others and
    turns itself into NaN (inf * 0)"""
    g = torch.tensor([1.0, 2.0, float("nan"), 3.0, 4.0])
    p = torch.nn.Parameter(torch.zeros(5))
    p.grad = g.clone()
    norm = torch.nn.utils.clip_grad_norm_([p], 40.0)
    assert torch.isnan(p.grad).all()
    c = O.clip_coef(np.float32(norm), 40.0)
    assert np.isnan(c)
    got = O.rmsprop_step(np.zeros(5), g.numpy(), np.zeros(5), None, None, c, 0.1, 0.99, 1e-8, 0.0, 0.0)[0]
    assert np.isnan(got["p"]).all()
    p = torch.nn.Parameter(torch.zeros(3))
    p.grad = torch.tensor([1.0, float("inf"), -2.0])
    norm = torch.nn.utils.clip_grad_norm_([p], 40.0)
    c = O.clip_coef(np.float32(norm), 40.0)
    assert c == 0.0
    got = O.adam_step(np.zeros(3), [1.0, np.inf, -2.0], np.zeros(3), np.zeros(3), c, 0.1, 0.9, 0.999, 1e-8, 0.0,
                      False, 1)[0]
    assert np.array_equal(np.isnan(got["g"]), torch.isnan(p.grad).numpy())
    assert np.array_equal(np.isnan(got["p"]), [False, True, False])
    # a NaN norm without a threshold: nothing is clipped, as clip_grad_norm_ is not called
    assert O.clip_coef(np.float32("nan"), -1.0) == 1.0
