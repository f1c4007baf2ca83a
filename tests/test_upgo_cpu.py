"""CPU: the float64 UPGO oracle against an independent closed form and two hand cases; the upgo_cost flag; the
tb_upgo_loss_f32 entry point in the header, the binding and its host-side checks; UPGO on / off in the graphed
learner's structure."""
import ctypes
import math
import os
import types

import numpy as np
import pytest
import torch

from tests import upgo_oracle as UO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A = 6


def _inputs(T, B, seed):
    rs = np.random.RandomState(seed)
    return dict(rewards=np.clip(2 * rs.randn(T, B), -1, 1), discounts=0.99 * (rs.rand(T, B) > 0.1),
                values=rs.randn(T, B), bootstrap=rs.randn(B))


@pytest.mark.parametrize("T,B,seed", [(1, 3, 0), (2, 4, 1), (17, 5, 2), (60, 3, 3)])
def test_recursion_matches_the_generalized_lambda_return(T, B, seed):
    kw = _inputs(T, B, seed)
    lam = UO.trace_switch(**kw)
    if T > 2:
        assert 0 < lam[1:].mean() < 1   # both branches are taken
    np.testing.assert_allclose(UO.returns(**kw), UO.return_general(**kw), rtol=1e-12, atol=1e-12)


def test_all_lambda_one_is_the_monte_carlo_return():
    T, B = 9, 4
    rs = np.random.RandomState(4)
    r, g = rs.rand(T, B), 0.9 * np.ones((T, B))
    v, bs = -10 * np.ones((T, B)), rs.randn(B)           # r + 0.9 V_{t+1} >= -10 for every r >= 0, V_{t+1} >= -11
    assert UO.trace_switch(r, g, v, bs)[1:].all()
    want = np.zeros((T, B))
    for t in range(T):
        acc, disc = np.zeros(B), np.ones(B)
        for k in range(t, T):
            acc += disc * r[k]
            disc = disc * g[k]
        want[t] = acc + disc * bs
    np.testing.assert_allclose(UO.returns(r, g, v, bs), want, rtol=1e-13)


def test_all_lambda_zero_is_the_one_step_return():
    T, B = 9, 4
    rs = np.random.RandomState(5)
    r, g = -rs.rand(T, B), 0.9 * np.ones((T, B))
    v, bs = 10 * np.ones((T, B)), 10 * np.ones(B)       # r + 9 < 10 for every r <= 0
    assert not UO.trace_switch(r, g, v, bs).any()
    v_next = np.concatenate([v[1:], bs[None]], 0)
    np.testing.assert_allclose(UO.returns(r, g, v, bs), r + g * v_next, rtol=1e-15)


def test_oracle_gradient_is_the_closed_form():
    T, B = 7, 5
    rs = np.random.RandomState(6)
    kw = _inputs(T, B, 6)
    tl, act, lr = rs.randn(T, B, A), rs.randint(0, A, size=(T, B)), 0.5 * rs.randn(T, B)
    w = rs.rand(B)
    o = UO.loss(tl, act, kw["rewards"], kw["discounts"], kw["values"], kw["bootstrap"], lr, 0.3, weights=w)
    pi = np.exp(tl - tl.max(-1, keepdims=True))
    pi /= pi.sum(-1, keepdims=True)
    want = 0.3 * (o["adv"] * w)[..., None] * (pi - np.eye(A)[act])
    np.testing.assert_allclose(o["grad_logits"], want, rtol=1e-12, atol=1e-15)
    rho_bar = np.minimum(np.exp(lr), 1.0)
    np.testing.assert_allclose(o["adv"], rho_bar * (o["G"] - kw["values"]), rtol=1e-15)


def _flags(v="absent"):
    f = types.SimpleNamespace(discounting=0.99)
    if v != "absent":
        f.upgo_cost = v
    return f


def test_flag_validation():
    from torchbeast_b200.learner import upgo_cost
    assert upgo_cost(_flags()) is None
    assert upgo_cost(_flags(None)) is None
    assert upgo_cost(_flags(0)) == 0.0
    assert upgo_cost(_flags(1.0)) == 1.0
    assert upgo_cost(_flags(np.float32(0.5))) == 0.5
    for bad in (-1e-9, -math.inf, math.inf, math.nan, "0.1", True, False, [0.1]):
        with pytest.raises(ValueError, match="upgo_cost"):
            upgo_cost(_flags(bad))


def test_symbol_is_in_header_and_binding():
    from torchbeast_b200 import _lib
    with open(os.path.join(ROOT, "include", "torchbeast_b200.h")) as f:
        assert "int tb_upgo_loss_f32(" in f.read()
    assert "tb_upgo_loss_f32" in _lib.declared_symbols()
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "tb_upgo_loss_f32")


def _call(**over):
    """tb_upgo_loss_f32 with never-dereferenced pointers: every case fails a host-side check before any launch."""
    from torchbeast_b200 import _lib
    P = ctypes.c_void_p(256)
    a = dict(tl=P, act=P, rw=P, done=P, disc=None, values=P, bootstrap=P, T=4, B=2, A=A, discounting=0.99,
             clip_rewards=1, clip_pg=1.0, hp=None, cw=None, task=None, mu=None, nu=None, K=0, log_rhos=P, beta=None,
             kl=None, cost=P, adv=P, out=P, losses=P, gl=P, ws=P, stream=None)
    a.update(over)
    rc = _lib.lib().tb_upgo_loss_f32(*a.values())
    return rc, _lib.lib().tb_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(cost=None), "must not be null"),
    (dict(out=None), "must not be null"),
    (dict(losses=None), "must not be null"),
    (dict(ws=None), "must not be null"),
    (dict(beta=ctypes.c_void_p(256)), "kl must not be null"),
    (dict(log_rhos=None), "null input pointer"),
    (dict(tl=None), "null input pointer"),
    (dict(done=None), "null input pointer"),
    (dict(adv=None), "upgo_adv must not be null"),
    (dict(A=0), "bad sizes"),
    (dict(T=-1), "bad sizes"),
    (dict(task=ctypes.c_void_p(256), K=2, mu=ctypes.c_void_p(256), nu=ctypes.c_void_p(256),
          cw=ctypes.c_void_p(256)), "column_weights are not supported with PopArt"),
    (dict(task=ctypes.c_void_p(256), K=65, mu=ctypes.c_void_p(256), nu=ctypes.c_void_p(256)), "num_tasks 65"),
    (dict(task=ctypes.c_void_p(256), K=2, mu=None, nu=ctypes.c_void_p(256)), "null PopArt pointer"),
    (dict(task=ctypes.c_void_p(256), K=2, mu=ctypes.c_void_p(256), nu=ctypes.c_void_p(256), T=0), "bad sizes"),
])
def test_host_side_checks(over, msg):
    rc, err = _call(**over)
    assert rc != 0 and msg in err, err


def test_upgo_on_off_and_cost_in_the_graphed_structure():
    from torchbeast_b200 import optim
    from torchbeast_b200.learner import GraphedLearner
    from torchbeast_b200.nets import AtariNet
    opt = optim.RMSprop(AtariNet((4, 84, 84), A, True, device="cpu"), lr=4.8e-4, eps=0.01)
    batch = {"done": torch.zeros(3, 2, dtype=torch.bool)}
    off = GraphedLearner.structure_of(opt, batch)
    assert GraphedLearner.structure_of(opt, batch, _flags()) == off
    assert GraphedLearner.structure_of(opt, batch, _flags(None)) == off
    on = GraphedLearner.structure_of(opt, batch, _flags(1.0))
    assert on != off
    # the cost is published per replay: any cost keeps the graph, 0 included
    for cost in (0.0, 0.25, 3.0):
        assert GraphedLearner.structure_of(opt, batch, _flags(cost)) == on
    both = _flags(1.0)
    both.trust_region_kl = 0.1
    assert GraphedLearner.structure_of(opt, batch, both) not in (on, off)
    with pytest.raises(ValueError, match="upgo_cost"):
        GraphedLearner.structure_of(opt, batch, _flags(-1.0))
