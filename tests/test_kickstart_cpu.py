"""CPU: the float64 kickstarting oracle against torch's kl_div and autograd (with -inf teacher logits); the
kickstart_cost flag; the tb_kickstart_loss_f32 entry point in the header, the binding and its host-side checks; the
Teacher attachment (state_dict keys, a bare net, the teacher checks); kickstarting on / off in the graphed learner's
structure."""
import ctypes
import math
import os
import types

import numpy as np
import pytest
import torch

from tests import kickstart_oracle as KO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A = 6


def _autograd(teacher, target, cost, weights):
    """loss and d loss / d target by torch.nn.functional.kl_div and autograd, float64."""
    s = torch.tensor(target, dtype=torch.float64, requires_grad=True)
    lt = torch.log_softmax(torch.tensor(teacher, dtype=torch.float64), -1)
    ls = torch.log_softmax(s, -1)
    rows = torch.nn.functional.kl_div(ls, lt, reduction="none", log_target=True).sum(-1)   # [T, B]
    total = cost * (rows * torch.tensor(weights, dtype=torch.float64)[None, :]).sum()
    total.backward()
    return rows.detach().numpy(), total.item(), s.grad.numpy()


@pytest.mark.parametrize("T,B,A_,seed", [(1, 1, 3, 0), (5, 4, 6, 1), (17, 3, 18, 2), (9, 7, 23, 3)])
def test_oracle_matches_kl_div_and_autograd(T, B, A_, seed):
    rs = np.random.RandomState(seed)
    teacher, target = 2 * rs.randn(T, B, A_), 2 * rs.randn(T, B, A_)
    w = rs.rand(B)
    rows, total, grad = _autograd(teacher, target, 0.7, w)
    o = KO.loss(teacher, target, 0.7, weights=w)
    np.testing.assert_allclose(o["kl"], rows, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(o["loss"], total, rtol=1e-12)
    np.testing.assert_allclose(o["grad_logits"], grad, rtol=1e-10, atol=1e-14)
    assert np.all(o["kl"] >= -1e-15)


def test_oracle_with_minus_inf_teacher_logits():
    rs = np.random.RandomState(4)
    T, B = 6, 5
    teacher, target = rs.randn(T, B, A), rs.randn(T, B, A)
    teacher[:, :, 0] = -np.inf          # an illegal action in every row
    teacher[2, 3, 1:4] = -np.inf        # a row with three of them
    o = KO.loss(teacher, target, 1.3)
    assert np.all(np.isfinite(o["kl"])) and np.all(np.isfinite(o["grad_logits"]))
    # the masked actions drop out: the KL is the one over the legal actions with the learner's full normaliser
    finite = np.where(np.isinf(teacher), -1e300, teacher)
    rows, total, grad = _autograd(finite, target, 1.3, np.ones(B))
    np.testing.assert_allclose(o["kl"], rows, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(o["grad_logits"], grad, rtol=1e-10, atol=1e-14)
    # the gradient on a masked action is cost * p_S(a) > 0: the learner is pushed off it
    assert np.all(o["grad_logits"][:, :, 0] > 0)


def test_identical_logits_give_zero():
    rs = np.random.RandomState(5)
    x = rs.randn(4, 3, A)
    o = KO.loss(x, x, 2.0)
    assert np.all(o["kl"] == 0) and np.all(o["grad_logits"] == 0) and o["loss"] == 0


def _flags(v="absent"):
    f = types.SimpleNamespace(discounting=0.99)
    if v != "absent":
        f.kickstart_cost = v
    return f


def test_flag_validation():
    from torchbeast_b200.kickstart import kickstart_cost
    assert kickstart_cost(_flags()) is None
    assert kickstart_cost(_flags(None)) is None
    assert kickstart_cost(_flags(0)) == 0.0
    assert kickstart_cost(_flags(1.0)) == 1.0
    assert kickstart_cost(_flags(np.float32(0.5))) == 0.5
    for bad in (-1e-9, -math.inf, math.inf, math.nan, "0.1", True, False, [0.1]):
        with pytest.raises(ValueError, match="kickstart_cost"):
            kickstart_cost(_flags(bad))


def test_symbol_is_in_header_and_binding():
    from torchbeast_b200 import _lib
    with open(os.path.join(ROOT, "include", "torchbeast_b200.h")) as f:
        assert "int tb_kickstart_loss_f32(" in f.read()
    assert "tb_kickstart_loss_f32" in _lib.declared_symbols()
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "tb_kickstart_loss_f32")


def _call(**over):
    """tb_kickstart_loss_f32 with never-dereferenced pointers: every case fails a host-side check before any launch."""
    from torchbeast_b200 import _lib
    P = ctypes.c_void_p(256)
    a = dict(teacher=P, target=P, T=4, B=2, A=A, cw=None, cost=P, out=P, losses=P, gl=P, ws=P, stream=None)
    a.update(over)
    rc = _lib.lib().tb_kickstart_loss_f32(*a.values())
    return rc, _lib.lib().tb_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(T=0), "bad sizes"),
    (dict(B=0), "bad sizes"),
    (dict(A=0), "bad sizes"),
    (dict(T=-1), "bad sizes"),
    (dict(teacher=None), "null input pointer"),
    (dict(target=None), "null input pointer"),
    (dict(cost=None), "must not be null"),
    (dict(out=None), "must not be null"),
    (dict(losses=None), "must not be null"),
    (dict(ws=None), "must not be null"),
])
def test_host_side_checks(over, msg):
    rc, err = _call(**over)
    assert rc != 0 and msg in err, err


def _atari(use_lstm=True, **kw):
    from torchbeast_b200.nets import AtariNet
    return AtariNet((4, 84, 84), kw.pop("num_actions", A), use_lstm, device="cpu", **kw)


def test_teacher_leaves_the_state_dict_keys_and_a_bare_net_raises():
    from torchbeast_b200 import _lib, learner
    from torchbeast_b200.kickstart import Teacher
    model, teacher_net = _atari(), _atari(use_lstm=False)
    keys = list(model.state_dict())
    model.teacher = Teacher(teacher_net)
    assert list(model.state_dict()) == keys
    assert not any(k.startswith("teacher") for k in model.state_dict())
    model.teacher = None
    bare = _atari()
    model.teacher = bare
    assert any(k.startswith("teacher.") for k in model.state_dict())   # what Teacher avoids
    for cost in (None, 1.0):
        flags = types.SimpleNamespace(kickstart_cost=cost)
        with pytest.raises(_lib.TorchBeastB200Error, match="Teacher"):
            learner.learn(flags, model, None, {}, (), None, None)


def test_cost_without_a_teacher_raises():
    from torchbeast_b200 import _lib, learner
    with pytest.raises(_lib.TorchBeastB200Error, match="no teacher"):
        learner.learn(types.SimpleNamespace(kickstart_cost=0.5), _atari(), None, {}, (), None, None)
    with pytest.raises(ValueError, match="kickstart_cost"):
        learner.learn(types.SimpleNamespace(kickstart_cost=-1.0), _atari(), None, {}, (), None, None)


def test_teacher_checks():
    from torchbeast_b200 import _lib
    from torchbeast_b200.kickstart import Teacher
    from torchbeast_b200.nets import ResNet
    model, actor = _atari(), _atari()
    Teacher(_atari(use_lstm=False, precision="bf16")).check(model, actor)          # any precision
    Teacher(_atari(num_tasks=3)).check(model, actor)                                # num_tasks: only logits are read
    Teacher(ResNet(A, True, device="cpu")).check(model, actor)                      # the other net, same observation
    with pytest.raises(_lib.TorchBeastB200Error, match="num_actions"):
        Teacher(_atari(num_actions=A + 1)).check(model, actor)
    with pytest.raises(_lib.TorchBeastB200Error, match="observation_shape"):
        Teacher(ResNet(A, device="cpu", observation_shape=(3, 64, 64))).check(model, actor)
    with pytest.raises(_lib.TorchBeastB200Error, match="learner model"):
        Teacher(model).check(model, actor)
    with pytest.raises(_lib.TorchBeastB200Error, match="actor model"):
        Teacher(actor).check(model, actor)
    shared = _atari()
    shared._flat = model._flat          # a net aliasing the learner's buffer
    with pytest.raises(_lib.TorchBeastB200Error, match="shares the learner model"):
        Teacher(shared).check(model, actor)
    with pytest.raises(_lib.TorchBeastB200Error, match="Teacher needs"):
        Teacher(torch.nn.Linear(2, 2))


def test_teacher_zero_state_is_kept_per_width():
    from torchbeast_b200.kickstart import Teacher
    t = Teacher(_atari())
    s4, s8 = t.initial_state(4), t.initial_state(8)
    assert t.initial_state(4) is s4 and s8 is not s4
    assert tuple(s4[0].shape) == (2, 4, 512 + A + 1) and all(torch.count_nonzero(x) == 0 for x in s4 + s8)
    assert Teacher(_atari(use_lstm=False)).initial_state(4) == ()


def test_kickstart_on_off_and_teacher_in_the_graphed_structure():
    from torchbeast_b200 import optim
    from torchbeast_b200.kickstart import Teacher
    from torchbeast_b200.learner import GraphedLearner
    model = _atari()
    opt = optim.RMSprop(model, lr=4.8e-4, eps=0.01)
    batch = {"done": torch.zeros(3, 2, dtype=torch.bool)}
    off = GraphedLearner.structure_of(opt, batch, _flags(), model)
    assert GraphedLearner.structure_of(opt, batch, _flags(None), model) == off
    model.teacher = Teacher(_atari(use_lstm=False))
    assert GraphedLearner.structure_of(opt, batch, _flags(None), model) == off     # attached, but off
    on = GraphedLearner.structure_of(opt, batch, _flags(1.0), model)
    assert on != off
    # the cost is published per replay: any cost keeps the graph, 0 included
    for cost in (0.0, 0.25, 3.0):
        assert GraphedLearner.structure_of(opt, batch, _flags(cost), model) == on
    # another teacher net is another graph; the same net in a new Teacher is not
    net = model.teacher.net
    model.teacher = Teacher(_atari(use_lstm=False))
    assert GraphedLearner.structure_of(opt, batch, _flags(1.0), model) not in (on, off)
    model.teacher = Teacher(net)
    assert GraphedLearner.structure_of(opt, batch, _flags(1.0), model) == on
    both = _flags(1.0)
    both.upgo_cost = 0.5
    assert GraphedLearner.structure_of(opt, batch, both, model) not in (on, off)
    with pytest.raises(ValueError, match="kickstart_cost"):
        GraphedLearner.structure_of(opt, batch, _flags(-1.0), model)
