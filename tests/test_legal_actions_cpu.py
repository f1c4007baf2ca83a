"""CPU: the float64 legal-action oracle against torch autograd of masked_fill(~legal, -inf) with an xlogy entropy (the
loss block, the trust region's KL, UPGO and kickstarting); the tb_mask_logits_f32 entry point and TB_MASKED_LOGIT in
the header, the binding and its host-side checks; the legal_actions learner leaf and its staging spec."""
import ctypes
import os
import re
import types

import numpy as np
import pytest
import torch

from tests import legal_actions_oracle as LO
from tests import upgo_oracle as UO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(T, B, A, seed):
    rs = np.random.RandomState(seed)
    legal = rs.rand(T, B, A) < 0.6
    legal[0, 0] = False                          # a row with no legal action: unmasked
    legal[min(1, T - 1), B - 1] = True           # an all-legal row
    actions = np.zeros((T, B), np.int64)
    for idx in np.ndindex(T, B):
        ok = np.flatnonzero(legal[idx]) if legal[idx].any() else np.arange(A)
        actions[idx] = rs.choice(ok)
    return dict(bl=2 * rs.randn(T, B, A), tl=2 * rs.randn(T, B, A), teacher=2 * rs.randn(T, B, A), legal=legal,
                actions=actions, rewards=np.clip(2 * rs.randn(T, B), -1, 1), discounts=0.99 * (rs.rand(T, B) > 0.2),
                values=rs.randn(T, B), bootstrap=rs.randn(B), weights=rs.rand(B))


def _masked(x, legal):
    """torch float64 logits with every illegal entry of a row that has a legal one set to -inf."""
    k = torch.from_numpy(LO.keep(legal))
    return torch.as_tensor(x, dtype=torch.float64).masked_fill(~k, float("-inf"))


def _torch_loss(d, beta, ent_cost=0.0006, bl_cost=0.5):
    """The loss block by torch autograd on masked_fill(-inf) logits, with the entropy as xlogy(p, p)."""
    tl = torch.tensor(d["tl"], dtype=torch.float64, requires_grad=True)
    k = torch.from_numpy(LO.keep(d["legal"]))
    lt = torch.log_softmax(tl.masked_fill(~k, float("-inf")), -1)
    lb = torch.log_softmax(_masked(d["bl"], d["legal"]), -1)
    pi = lt.exp()
    # xlogy(p, p) is 0 at p = 0; its second argument is 1 there so that no 0 * (-inf) enters the gradient either
    kl = (torch.xlogy(pi, pi.masked_fill(~k, 1.0)) - pi * lb.masked_fill(~k, 0.0)).sum(-1)
    mask = torch.ones_like(kl, dtype=torch.bool) if beta is None else kl.detach() <= beta
    a = torch.from_numpy(d["actions"])[..., None]
    tlp, blp = lt.gather(-1, a)[..., 0], lb.gather(-1, a)[..., 0]
    w = torch.from_numpy(d["weights"])
    with torch.no_grad():
        rho = torch.where(mask, torch.exp(tlp - blp), torch.zeros(()))
        r, g = torch.from_numpy(d["rewards"]), torch.from_numpy(d["discounts"])
        v, bs = torch.from_numpy(d["values"]), torch.from_numpy(d["bootstrap"])
        rho_bar, cs = rho.clamp(max=1.0), rho.clamp(max=1.0)
        v_next = torch.cat([v[1:], bs[None]])
        deltas = rho_bar * (r + g * v_next - v)
        acc, vs = torch.zeros_like(bs), torch.zeros_like(v)
        for t in range(v.shape[0] - 1, -1, -1):
            acc = deltas[t] + g[t] * cs[t] * acc
            vs[t] = acc
        vs = vs + v
        pg_adv = rho.clamp(max=1.0) * (r + g * torch.cat([vs[1:], bs[None]]) - v)
    ent_row = torch.xlogy(pi, pi.masked_fill(~k, 1.0)).sum(-1)
    pg = (-tlp * pg_adv * w).sum()
    ent = ent_cost * (ent_row * w).sum()
    base = bl_cost * (0.5 * (vs - v) ** 2 * w).sum()
    total = pg + base + ent
    total.backward()
    return dict(kl=kl.detach().numpy(), mask=mask.numpy(), log_rhos=(tlp - blp).detach().numpy(), vs=vs.numpy(),
                losses=np.array([pg.item(), base.item(), ent.item(), total.item()]), grad_logits=tl.grad.numpy())


@pytest.mark.parametrize("T,B,A,seed,beta", [(5, 4, 6, 0, None), (7, 3, 18, 1, 0.3), (4, 5, 2, 2, None),
                                             (6, 2, 23, 3, 0.1)])
def test_oracle_loss_matches_masked_fill_autograd(T, B, A, seed, beta):
    d = _inputs(T, B, A, seed)
    want = _torch_loss(d, beta)
    o = LO.loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["discounts"], d["values"], d["bootstrap"], d["legal"],
                beta=beta, weights=d["weights"])
    assert np.array_equal(o["mask"], want["mask"])
    for k in ("kl", "log_rhos", "vs", "losses", "grad_logits"):
        np.testing.assert_allclose(o[k], want[k], rtol=1e-11, atol=1e-13, err_msg=k)
    # the dropped entries get gradient 0, not NaN; the oracle reaches it without any -inf
    assert np.all(np.isfinite(o["grad_logits"]))
    assert np.all(o["grad_logits"][~LO.keep(d["legal"])] == 0)


@pytest.mark.parametrize("T,B,A,seed", [(6, 3, 6, 4), (5, 4, 18, 5)])
def test_oracle_upgo_and_kickstart_match_masked_fill_autograd(T, B, A, seed):
    d = _inputs(T, B, A, seed)
    k = torch.from_numpy(LO.keep(d["legal"]))
    log_rhos = np.random.RandomState(seed).randn(T, B) * 0.3
    # UPGO: cost * sum w (-log pi(a)) adv, by autograd through the masked log-softmax
    o = LO.upgo(d["tl"], d["actions"], d["rewards"], d["discounts"], d["values"], d["bootstrap"], log_rhos, d["legal"],
                0.7, weights=d["weights"])
    tl = torch.tensor(d["tl"], dtype=torch.float64, requires_grad=True)
    lt = torch.log_softmax(tl.masked_fill(~k, float("-inf")), -1)
    lpa = lt.gather(-1, torch.from_numpy(d["actions"])[..., None])[..., 0]
    G = UO.returns(d["rewards"], d["discounts"], d["values"], d["bootstrap"])
    adv = np.minimum(np.exp(log_rhos), 1.0) * (G - d["values"])
    total = 0.7 * (-lpa * torch.from_numpy(adv) * torch.from_numpy(d["weights"])).sum()
    total.backward()
    np.testing.assert_allclose(o["loss"], total.item(), rtol=1e-12)
    np.testing.assert_allclose(o["grad_logits"], tl.grad.numpy(), rtol=1e-10, atol=1e-14)
    # kickstarting: torch's kl_div on the two masked log-softmaxes
    o = LO.kickstart(d["teacher"], d["tl"], d["legal"], 1.3, weights=d["weights"])
    s = torch.tensor(d["tl"], dtype=torch.float64, requires_grad=True)
    ls = torch.log_softmax(s.masked_fill(~k, float("-inf")), -1)
    lt = torch.log_softmax(_masked(d["teacher"], d["legal"]), -1)
    rows = torch.nn.functional.kl_div(ls, lt, reduction="none", log_target=True).nan_to_num(0.0).sum(-1)
    total = 1.3 * (rows * torch.from_numpy(d["weights"])[None, :]).sum()
    total.backward()
    np.testing.assert_allclose(o["kl"], rows.detach().numpy(), rtol=1e-11, atol=1e-13)
    np.testing.assert_allclose(o["loss"], total.item(), rtol=1e-12)
    np.testing.assert_allclose(o["grad_logits"], np.nan_to_num(s.grad.numpy()), rtol=1e-10, atol=1e-14)


def test_mask_restatement_rules():
    x = np.arange(12, dtype=np.float32).reshape(3, 4)
    legal = np.array([[1, 0, 1, 0], [0, 0, 0, 0], [1, 1, 0, 1]], bool)
    out = LO.mask_logits(x, legal)
    fmin = np.finfo(np.float32).min
    assert np.array_equal(out, [[0, fmin, 2, fmin], [4, 5, 6, 7], [8, 9, fmin, 11]])
    out = LO.mask_logits(x, legal, actions=np.array([1, 3, 7]))   # illegal; a row with no legal action; out of range
    assert np.all(np.isnan(out[0])) and np.array_equal(out[1:], [[4, 5, 6, 7], [8, 9, fmin, 11]])


def test_header_declares_the_entry_and_the_sentinel():
    from torchbeast_b200 import _lib
    from torchbeast_b200.legal_actions import MASKED_LOGIT
    with open(os.path.join(ROOT, "include", "torchbeast_b200.h")) as f:
        text = f.read()
    assert "int tb_mask_logits_f32(const float* in, float* out, const uint8_t* legal, const int64_t* actions, " in text
    m = re.search(r"#define TB_MASKED_LOGIT \((\S+)F\)", text)
    assert m is not None
    assert np.float32(float(m.group(1))) == np.float32(torch.finfo(torch.float32).min) == np.float32(MASKED_LOGIT)
    assert np.isfinite(np.float32(float(m.group(1))))
    assert "tb_mask_logits_f32" in _lib.declared_symbols()
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "tb_mask_logits_f32")


def _call(**over):
    """tb_mask_logits_f32 with never-dereferenced pointers: every case fails a host-side check before any launch."""
    from torchbeast_b200 import _lib
    P = ctypes.c_void_p(256)
    a = dict(inp=P, out=P, legal=P, actions=None, N=4, A=6, fill=0.0, stream=None)
    a.update(over)
    rc = _lib.lib().tb_mask_logits_f32(*a.values())
    return rc, _lib.lib().tb_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(inp=None), "null pointer"),
    (dict(out=None), "null pointer"),
    (dict(legal=None), "null pointer"),
    (dict(A=0), "A must be at least 1"),
    (dict(A=-3), "A must be at least 1"),
    (dict(N=-1), "negative size"),
    (dict(N=2 ** 62, A=4), "size overflow"),
])
def test_host_side_checks(over, msg):
    rc, err = _call(**over)
    assert rc != 0 and msg in err, err


def test_zero_rows_is_a_no_op_success():
    rc, err = _call(N=0, inp=None, out=None, legal=None)
    assert rc == 0, err


def test_leaf_is_a_learner_key_and_a_staging_leaf():
    from torchbeast_b200 import staging
    from torchbeast_b200.learner import GraphedLearner
    from torchbeast_b200.replay import ReplayBuffer  # noqa: F401
    assert "legal_actions" in GraphedLearner.KEYS
    assert len(GraphedLearner.KEYS) + 2 <= 16       # TB_REPLAY_MAX_LEAVES, with an LSTM's two state leaves
    T, B, A = 80, 32, 6
    spec = staging.spec_for(T, B, A, extra=(("legal_actions", (T + 1, B, A), torch.bool),))
    assert spec["legal_actions"] == ((T + 1, B, A), torch.bool)
    assert spec["policy_logits"] == ((T + 1, B, A), torch.float32)


def _batch(T=3, B=2, A=6, **legal):
    b = dict(frame=torch.zeros(T + 1, B, 4, 84, 84, dtype=torch.uint8), reward=torch.zeros(T + 1, B),
              done=torch.zeros(T + 1, B, dtype=torch.bool), policy_logits=torch.zeros(T + 1, B, A),
              action=torch.zeros(T + 1, B, dtype=torch.int64))
    if legal:
        b["legal_actions"] = legal["t"]
    return b


@pytest.mark.parametrize("leaf,msg", [
    (torch.ones(4, 2, 6, dtype=torch.float32), "must be bool or uint8"),
    (torch.ones(4, 2, 6, dtype=torch.int64), "must be bool or uint8"),
    (torch.ones(3, 2, 6, dtype=torch.bool), "(T+1, B, A) = (4, 2, 6)"),
    (torch.ones(4, 2, 5, dtype=torch.uint8), "(T+1, B, A) = (4, 2, 6)"),
    (torch.ones(4, 2, dtype=torch.bool), "(T+1, B, A) = (4, 2, 6)"),
    (torch.ones(4, 2, 6, dtype=torch.bool, device="meta"), "is on meta"),
])
def test_learn_validates_the_leaf_before_anything_is_staged(leaf, msg):
    from torchbeast_b200 import learner
    from torchbeast_b200._lib import TorchBeastB200Error

    class Model:  # learn() must raise before it touches the model, the optimizer or the device
        def __getattr__(self, name):
            raise AssertionError("learn() read model.%s before checking legal_actions" % name)

    with pytest.raises(TorchBeastB200Error) as e:
        learner.learn(types.SimpleNamespace(), Model(), None, _batch(t=leaf), (), None, None)
    assert msg in str(e.value)


def test_valid_leaf_passes_the_check():
    from torchbeast_b200.legal_actions import check_leaf
    check_leaf(_batch())
    check_leaf(_batch(t=torch.ones(4, 2, 6, dtype=torch.bool)))
    check_leaf(_batch(t=torch.ones(4, 2, 6, dtype=torch.uint8)))
