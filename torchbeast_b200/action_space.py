"""Multi-discrete (factored) action spaces: an action is a tuple of D independent choices (gym's MultiDiscrete).

A net built with `num_actions=(A_1, ..., A_D)` has a policy that is a product of D categoricals: its policy logits are
[T, B, A_1 + ... + A_D], component k owning the columns [off_k, off_k + A_k), and its actions (and `last_action`) are
int64 [T, B, D].  log pi(a) = sum_k log pi_k(a_k), and the entropy and the trust region's KL are sums over components
too (include/torchbeast_b200.h, "multi-discrete (factored) action spaces", states the rules).  An int `num_actions` is
the flat policy, unchanged.

UPGO, kickstarting and legal-action masks take flat rows only; a learner with a factored space raises for them before
anything is launched (check_learner).
"""
import ctypes

import torch

from torchbeast_b200 import _lib

MAX_COMPONENTS = 16  # TB_MAX_ACTION_COMPONENTS


class CActionSpace(ctypes.Structure):
    """tb_action_space, the host struct every factored entry point takes."""
    _fields_ = [("num_components", ctypes.c_int32), ("dims", ctypes.c_int32 * MAX_COMPONENTS)]


def dims_of(num_actions):
    """The component sizes (A_1, ..., A_D) of a tuple or list `num_actions`, checked (1 <= D <= 16, every A_k an int
    >= 1); None for an int (a flat policy)."""
    if isinstance(num_actions, (tuple, list)):
        dims = tuple(num_actions)
        if not 1 <= len(dims) <= MAX_COMPONENTS or any(
                isinstance(a, bool) or not isinstance(a, int) or a < 1 for a in dims):
            raise _lib.TorchBeastB200Error("a factored num_actions must be a tuple of 1 to %d ints >= 1, got %r"
                                           % (MAX_COMPONENTS, num_actions))
        return dims
    return None


def width(num_actions):
    """The policy-logit width: num_actions itself, or the sum of a tuple's component sizes."""
    dims = dims_of(num_actions)
    return num_actions if dims is None else sum(dims)


def c_space(dims):
    """The tb_action_space of `dims`, passed by reference to the C entry points."""
    s = CActionSpace()
    s.num_components = len(dims)
    for k, a in enumerate(dims):
        s.dims[k] = a
    return s


def dims_of_model(model):
    """A model's component sizes, or None for a flat policy."""
    return getattr(model, "action_dims", None)


def greedy(logits, dims):
    """The eval-mode action of a factored policy: argmax per segment, int64 [T, B, D]."""
    return torch.stack([seg.argmax(-1) for seg in logits.detach().split(dims, dim=-1)], dim=-1)


def multinomial(logits, dims):
    """torch.multinomial per segment, int64 [T, B, D]: what a factored net samples without an ActionSampler."""
    T, B = logits.shape[:2]
    return torch.stack([torch.multinomial(torch.softmax(seg.reshape(T * B, -1), dim=1), num_samples=1).view(T, B)
                        for seg in logits.detach().split(dims, dim=-1)], dim=-1)


def check_learner(model, flags, batch, teacher):
    """Raises, before anything is staged or launched, when a learner with a factored space is asked for what takes
    flat rows only: UPGO (flags.upgo_cost), kickstarting (flags.kickstart_cost), a legal_actions leaf, or a teacher whose
    space differs from the learner's."""
    dims = dims_of_model(model)
    if teacher is not None and dims_of_model(teacher.net) != dims:
        raise _lib.TorchBeastB200Error("the teacher's action space %r differs from the learner's %r"
                                       % (dims_of_model(teacher.net) or teacher.net.num_actions,
                                          dims or model.num_actions))
    if dims is None:
        return
    not_built = []
    if getattr(flags, "upgo_cost", None) is not None:
        not_built.append("UPGO (flags.upgo_cost)")
    if getattr(flags, "kickstart_cost", None) is not None:
        not_built.append("kickstarting (flags.kickstart_cost)")
    if isinstance(batch, dict) and batch.get("legal_actions") is not None:
        not_built.append("legal-action masks (a legal_actions leaf)")
    if not_built:
        raise _lib.TorchBeastB200Error("%s: not built for a factored action space %r" % (", ".join(not_built), dims))
