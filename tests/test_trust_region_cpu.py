"""CPU: the float64 trust-region oracle against the reference V-trace and losses, its limits and gradients; the
trust_region_kl flag; the two entry points in the library; trust on / off in the graphed learner's structure."""
import ctypes
import math
import types

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests import trust_region_oracle as TO

A = 6


def _inputs(T, B, seed, A=A):
    rs = np.random.RandomState(seed)
    return dict(behavior_logits=rs.randn(T, B, A), target_logits=rs.randn(T, B, A),
                actions=rs.randint(0, A, size=(T, B)), rewards=np.clip(2 * rs.randn(T, B), -1, 1),
                discounts=0.99 * (rs.rand(T, B) > 0.1), values=rs.randn(T, B), bootstrap=rs.randn(B))


def _reference(kw, bc=0.5, ec=0.0006):
    t = {k: torch.from_numpy(np.asarray(v)) for k, v in kw.items()}
    vs, pg_adv, lr, blp, tlp = LT.vtrace_from_logits_torch(t["behavior_logits"], t["target_logits"], t["actions"],
                                                          t["discounts"], t["rewards"], t["values"], t["bootstrap"])
    pg, bl, en = LT.impala_losses_torch(t["target_logits"], t["actions"], pg_adv, vs, t["values"], bc, ec)
    return vs.numpy(), pg_adv.numpy(), lr.numpy(), np.array([pg.item(), bl.item(), en.item()])


@pytest.mark.parametrize("beta", [None, math.inf])
def test_infinite_beta_is_the_reference_vtrace_and_losses(beta):
    kw = _inputs(13, 5, 1)
    o = TO.loss(**kw, beta=beta)
    vs, pg_adv, lr, losses = _reference(kw)
    assert o["mask"].all() and o["trusted"] == 13 * 5
    np.testing.assert_allclose(o["vs"], vs, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(o["pg_adv"], pg_adv, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(o["log_rhos"], lr, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(o["losses"][:3], losses, rtol=1e-12, atol=1e-12)


def test_every_row_untrusted_leaves_baseline_and_entropy_only():
    kw = _inputs(9, 4, 2)
    ec = 0.01
    o = TO.loss(**kw, beta=-1.0, entropy_cost=ec)   # kl >= 0 > beta: no row is trusted
    assert not o["mask"].any() and o["trusted"] == 0
    assert np.all(o["pg_adv"] == 0) and o["losses"][0] == 0
    np.testing.assert_array_equal(o["vs"], kw["values"])
    np.testing.assert_array_equal(o["grad_values"], np.zeros_like(kw["values"]))
    lt = TO.log_softmax(kw["target_logits"])
    pi = np.exp(lt)
    entropy_only = ec * pi * (lt - (pi * lt).sum(-1, keepdims=True))
    np.testing.assert_allclose(o["grad_logits"], entropy_only, rtol=1e-13, atol=1e-15)
    # the unmasked quantities do not change
    full = TO.loss(**kw, beta=None, entropy_cost=ec)
    np.testing.assert_array_equal(o["log_rhos"], full["log_rhos"])
    np.testing.assert_array_equal(o["kl"], full["kl"])


def test_kl_is_zero_for_identical_policies_and_positive_otherwise():
    kw = _inputs(5, 3, 3)
    assert np.all(TO.policy_kl(kw["target_logits"], kw["target_logits"]) == 0)
    assert np.all(TO.policy_kl(kw["behavior_logits"], kw["target_logits"]) > 0)
    o = TO.loss(**dict(kw, behavior_logits=kw["target_logits"]), beta=0.0)
    assert o["mask"].all()


@pytest.mark.parametrize("weighted", [False, True])
def test_oracle_gradients_match_autograd_with_the_mask_held_constant(weighted):
    kw = _inputs(11, 6, 4)
    bc, ec = 0.5, 0.01
    beta = float(np.median(TO.policy_kl(kw["behavior_logits"], kw["target_logits"])))
    w = np.random.RandomState(5).rand(6) if weighted else None
    o = TO.loss(**kw, beta=beta, baseline_cost=bc, entropy_cost=ec, weights=w)
    assert 0 < o["trusted"] < 11 * 6
    tl = torch.tensor(kw["target_logits"], requires_grad=True)
    v = torch.tensor(kw["values"], requires_grad=True)
    lp = torch.log_softmax(tl, -1)
    lpa = lp.gather(-1, torch.from_numpy(kw["actions"])[..., None])[..., 0]
    vs, adv = torch.from_numpy(o["vs"]), torch.from_numpy(o["pg_adv"])     # constants: no gradient through kl or m
    wt = torch.ones(6, dtype=torch.float64) if w is None else torch.from_numpy(w)
    total = ((-lpa * adv + bc * 0.5 * (vs - v) ** 2 + ec * (lp.exp() * lp).sum(-1)) * wt).sum()
    total.backward()
    np.testing.assert_allclose(o["losses"][3], total.item(), rtol=1e-13)
    np.testing.assert_allclose(o["grad_logits"], tl.grad.numpy(), rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(o["grad_values"], v.grad.numpy(), rtol=1e-10, atol=1e-13)


def test_mask_cuts_the_trace_at_an_untrusted_step():
    kw = _inputs(6, 1, 6)
    mask = np.ones((6, 1), bool)
    mask[3] = False
    o = TO.loss(**kw, mask=mask)
    full = TO.loss(**kw)
    # rows after the cut do not see it; row 3 keeps only the discounted trace of later rows through c_3 = 0: vs_3 = V_3
    np.testing.assert_array_equal(o["vs"][4:], full["vs"][4:])
    assert o["vs"][3, 0] == kw["values"][3, 0] and o["pg_adv"][3, 0] == 0
    # earlier rows still bootstrap from vs_3 through their own TD errors
    assert not np.allclose(o["vs"][:3], full["vs"][:3])


def _flags(v="absent"):
    f = types.SimpleNamespace(discounting=0.99)
    if v != "absent":
        f.trust_region_kl = v
    return f


def test_flag_validation():
    from torchbeast_b200.learner import trust_region_kl
    assert trust_region_kl(_flags()) is None
    assert trust_region_kl(_flags(None)) is None
    assert trust_region_kl(_flags(0)) == 0.0
    assert trust_region_kl(_flags(0.25)) == 0.25
    assert trust_region_kl(_flags(np.float32(0.5))) == 0.5
    assert trust_region_kl(_flags(math.inf)) == math.inf
    for bad in (-1e-9, -math.inf, math.nan, "0.1", True, [0.1]):
        with pytest.raises(ValueError, match="trust_region_kl"):
            trust_region_kl(_flags(bad))


def test_loss_entry_point_is_exported_and_checks_trust_outputs():
    from torchbeast_b200 import _lib
    h = ctypes.CDLL(_lib.LIB_PATH)
    name = "tb_impala_loss_f32"
    assert hasattr(h, name)
    assert name in _lib.declared_symbols()
    P = ctypes.c_void_p(256)  # never dereferenced: every call below fails its host-side checks before a launch
    for kl, sums in ((None, P), (P, None)):
        args = ([None] * 8 + [4, 2, A, 0.99, 0.5, 0.0006, 1, 1.0, 1.0] + [None] * 5 + [0, None, P, kl, sums]
                + [None] * 5 + [P, None, None, 1, P, None])
        assert getattr(_lib.lib(), name)(*args) != 0
        assert b"kl_out/trust_out must not be null" in _lib.lib().tb_last_error()


def test_trust_on_off_selects_another_graph():
    from torchbeast_b200 import optim
    from torchbeast_b200.learner import GraphedLearner
    from torchbeast_b200.nets import AtariNet
    opt = optim.RMSprop(AtariNet((4, 84, 84), A, True, device="cpu"), lr=4.8e-4, eps=0.01)
    batch = {"done": torch.zeros(3, 2, dtype=torch.bool)}
    off = GraphedLearner.structure_of(opt, batch)
    assert GraphedLearner.structure_of(opt, batch, _flags()) == off
    assert GraphedLearner.structure_of(opt, batch, _flags(None)) == off
    on = GraphedLearner.structure_of(opt, batch, _flags(0.1))
    assert on != off
    # beta itself is published per replay: any beta keeps the graph
    for beta in (0.0, 3.0, math.inf):
        assert GraphedLearner.structure_of(opt, batch, _flags(beta)) == on
    with pytest.raises(ValueError):
        GraphedLearner.structure_of(opt, batch, _flags(-1.0))
