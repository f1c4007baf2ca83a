"""CPU: the float64 restatement of csrc/vtrace.cu in tests/loss_oracle.py against the other restatements of the same
arithmetic - oracle/vtrace_np.py (float64, pinned to the reference by tests/test_oracle_golden.py), oracle/vtrace_c.c
(float32, through oracle/c_api.py) and torch float64 autograd for the gradients - for every clip setting (None, 0,
finite, +inf; NaN and negative as None), with done and with discounts.  The GPU kernel tests trust this restatement and
its magnitudes, so both are checked here: another float64 computation must lie within the float64 bound, and the
float32 C restatement within the float32 bound."""
import numpy as np
import pytest
import torch

from oracle import c_api
from oracle import vtrace_np as VO
from tests import loss_oracle as LO

# exact in float32, so that every restatement holds the same scalars
GAMMA, BC, EC = 0.75, 0.5, 0.0625
CLIPS = [(None, None), (0.0, 0.0), (1.0, 1.0), (3.75, 2.25), (0.5, 1.5), (np.inf, np.inf)]
SHAPES = [(1, 1, 2), (7, 5, 6), (40, 9, 11), (3, 33, 1)]


def _inputs(T, B, A, seed):
    rs = np.random.RandomState(seed)
    return dict(bl=rs.randn(T, B, A).astype(np.float32), tl=rs.randn(T, B, A).astype(np.float32),
                a=rs.randint(0, A, size=(T, B)), r=(2 * rs.randn(T, B)).astype(np.float32), done=rs.rand(T, B) < 0.1,
                v=rs.randn(T, B).astype(np.float32), bs=rs.randn(B).astype(np.float32))


def _within(got, want, mag, u, what):
    err = np.abs(np.asarray(got, np.float64) - want)
    tol = LO.bound(mag, u)
    assert np.all(err <= tol), "%s: %.3g of the bound" % (what, float((err / (tol + 1e-300)).max()))


def _vo_clip(c):
    return None if c is None else float(c)


@pytest.mark.parametrize("clips", CLIPS, ids=[str(c) for c in CLIPS])
@pytest.mark.parametrize("T,B,A", SHAPES)
def test_loss_matches_vtrace_np(T, B, A, clips):
    x = _inputs(T, B, A, T * 100 + B + A)
    o = LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"], done=x["done"], discounting=GAMMA,
                       baseline_cost=BC, entropy_cost=EC, clip_rho=clips[0], clip_pg_rho=clips[1])
    ref = VO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["done"], x["v"], x["bs"], discounting=GAMMA,
                         baseline_cost=BC, entropy_cost=EC, clip_rho_threshold=_vo_clip(clips[0]),
                         clip_pg_rho_threshold=_vo_clip(clips[1]), dtype=np.float64)
    for name, want in (("vs", ref.vtrace.vs), ("pg_adv", ref.vtrace.pg_advantages), ("log_rhos", ref.vtrace.log_rhos),
                       ("target_alp", ref.vtrace.target_action_log_probs),
                       ("behavior_alp", ref.vtrace.behavior_action_log_probs), ("grad_logits", ref.grad_logits),
                       ("grad_values", ref.grad_values)):
        _within(o[name], want, o["mag_" + name], LO.U64, name)
    _within(o["losses"], [ref.pg_loss, ref.baseline_loss, ref.entropy_loss, ref.total_loss], o["mag_losses"], LO.U64,
            "losses")


@pytest.mark.parametrize("clips", CLIPS, ids=[str(c) for c in CLIPS])
@pytest.mark.parametrize("T,B,A", SHAPES)
def test_discounts_give_the_done_path(T, B, A, clips):
    x = _inputs(T, B, A, T + 7 * B + A)
    kw = dict(discounting=GAMMA, baseline_cost=BC, entropy_cost=EC, clip_rho=clips[0], clip_pg_rho=clips[1])
    a = LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"], done=x["done"], **kw)
    b = LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"],
                       discounts=np.where(x["done"], 0.0, GAMMA).astype(np.float32), **kw)
    for k, v in a.items():
        assert np.array_equal(v, b[k]), k


@pytest.mark.parametrize("clips", CLIPS, ids=[str(c) for c in CLIPS])
def test_scan_matches_vtrace_np_and_the_float32_c_restatement(clips):
    T, B = 50, 7
    rs = np.random.RandomState(3)
    lr = (0.8 * rs.randn(T, B)).astype(np.float32)
    g = (GAMMA * (rs.rand(T, B) > 0.1)).astype(np.float32)
    r, v, bs = rs.randn(T, B).astype(np.float32), rs.randn(T, B).astype(np.float32), rs.randn(B).astype(np.float32)
    o = LO.scan(lr, g, r, v, bs, *clips)
    ref = VO.from_importance_weights(lr, g, r, v, bs, _vo_clip(clips[0]), _vo_clip(clips[1]), dtype=np.float64)
    _within(o["vs"], ref.vs, o["mag_vs"], LO.U64, "vs")
    _within(o["pg_adv"], ref.pg_advantages, o["mag_pg"], LO.U64, "pg_adv")
    cvs, cpg = c_api.vtrace_scan(lr, g, r, v, bs, *clips)
    _within(cvs, o["vs"], o["mag_vs"], LO.U32, "vs (float32 C)")
    _within(cpg, o["pg_adv"], o["mag_pg"], LO.U32, "pg_adv (float32 C)")
    # a NaN or negative threshold means no clipping
    if clips == (None, None):
        for c in (np.nan, -1.0):
            o2 = LO.scan(lr, g, r, v, bs, c, c)
            assert np.array_equal(o2["vs"], o["vs"]) and np.array_equal(o2["pg_adv"], o["pg_adv"])


@pytest.mark.parametrize("T,B,A", SHAPES)
def test_loss_within_the_float32_bound_of_the_c_restatement(T, B, A):
    x = _inputs(T, B, A, 11 * T + B)
    o = LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"], done=x["done"], discounting=GAMMA,
                       baseline_cost=BC, entropy_cost=EC)
    c = c_api.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["done"], x["v"], x["bs"], discounting=GAMMA,
                          baseline_cost=BC, entropy_cost=EC)
    for name, key in (("vs", "vs"), ("pg_advantages", "pg_adv"), ("grad_logits", "grad_logits"),
                      ("grad_values", "grad_values")):
        _within(c[name], o[key], o["mag_" + key], LO.U32, name)
    _within(c["losses"], o["losses"][:3], o["mag_losses"][:3], LO.U32, "losses")


@pytest.mark.parametrize("clips", CLIPS, ids=[str(c) for c in CLIPS])
@pytest.mark.parametrize("T,B,A", SHAPES)
def test_gradients_match_torch_autograd(T, B, A, clips):
    """d total / d target logits and d values with vs and pg_adv held constant, as the reference's backward holds them"""
    x = _inputs(T, B, A, 5 * T + B + A)
    x["tl"][0, 0, (x["a"][0, 0] + 1) % A] = LO.MASKED_LOGIT if A > 1 else x["tl"][0, 0, 0]
    o = LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"], done=x["done"], discounting=GAMMA,
                       baseline_cost=BC, entropy_cost=EC, clip_rho=clips[0], clip_pg_rho=clips[1])
    tl = torch.tensor(x["tl"], dtype=torch.float64, requires_grad=True)
    v = torch.tensor(x["v"], dtype=torch.float64, requires_grad=True)
    lsm = torch.log_softmax(tl, -1)
    lpa = lsm.gather(-1, torch.from_numpy(x["a"])[..., None])[..., 0]
    vs, adv = torch.from_numpy(o["vs"]), torch.from_numpy(o["pg_adv"])
    p = lsm.exp()
    ent = torch.where(p > 0, p * lsm, torch.zeros_like(p)).sum(-1)
    total = (-lpa * adv).sum() + BC * 0.5 * ((vs - v) ** 2).sum() + EC * ent.sum()
    total.backward()
    _within(o["grad_logits"], tl.grad.numpy(), o["mag_grad_logits"], LO.U64, "grad_logits")
    _within(o["grad_values"], v.grad.numpy(), o["mag_grad_values"], LO.U64, "grad_values")
    _within(o["losses"][3], total.item(), o["mag_losses"][3], LO.U64, "total")


def test_action_log_probs_and_standalone_losses_match_torch():
    rs = np.random.RandomState(9)
    for A in (1, 2, 6, 19):
        x = rs.randn(40, A) * 3
        x[::5] += 1e4
        x[1::7] = 0.5
        a = rs.randint(0, A, size=40)
        adv = rs.randn(40)
        t = torch.tensor(x, requires_grad=True)
        lsm = torch.log_softmax(t, -1)
        lp, mag = LO.action_log_probs(x, a)
        _within(lp, lsm.gather(-1, torch.from_numpy(a)[:, None])[:, 0].detach().numpy(), mag, LO.U64, "alp")
        e = LO.entropy_loss(x, LO.U64)
        ent = (lsm.exp() * lsm).sum()
        (gt,) = torch.autograd.grad(ent, t, retain_graph=True)
        _within(e["out"], ent.item(), e["mag_out"], LO.U64, "entropy")
        _within(e["grad"], gt.numpy(), e["mag_grad"], LO.U64, "entropy grad")
        if A == 1:
            assert e["out"] == 0 and not e["grad"].any()
        pg = LO.pg_loss(x, a, adv, LO.U64)
        pgt = (-lsm.gather(-1, torch.from_numpy(a)[:, None])[:, 0] * torch.from_numpy(adv)).sum()
        (gt,) = torch.autograd.grad(pgt, t)
        _within(pg["out"], pgt.item(), pg["mag_out"], LO.U64, "pg")
        _within(pg["grad"], gt.numpy(), pg["mag_grad"], LO.U64, "pg grad")
    b = LO.baseline_loss(adv)
    assert b["out"] == 0.5 * float((adv ** 2).sum()) and np.array_equal(b["grad"], adv)


@pytest.mark.parametrize("mistake", LO.MISTAKES)
def test_every_mistake_changes_the_result(mistake):
    """each mistake the GPU tests show their bounds reject moves this restatement at the shapes they use (the ratios
    themselves are asserted there, beside the kernel's own error)"""
    T, B, A = (80, 960, 6) if mistake == "fp32_sums" else (20, 9, 6)
    x = _inputs(T, B, A, 1)
    kw = dict(done=x["done"], discounting=GAMMA, baseline_cost=BC, entropy_cost=EC, clip_rho=2.0, clip_pg_rho=0.5)
    o = LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"], **kw)
    m = LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"], mistake=mistake, **kw)
    assert any(not np.array_equal(o[k], m[k]) for k in o if not k.startswith("mag_")), mistake
