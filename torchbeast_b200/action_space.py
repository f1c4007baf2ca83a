"""Multi-discrete (factored) action spaces: an action is a tuple of D independent choices (gym's MultiDiscrete).

A net built with `num_actions=(A_1, ..., A_D)` has a policy that is a product of D categoricals: its policy logits are
[T, B, A_1 + ... + A_D], component k owning the columns [off_k, off_k + A_k), and its actions (and `last_action`) are
int64 [T, B, D].  log pi(a) = sum_k log pi_k(a_k), and the entropy and the trust region's KL are sums over components
too (include/torchbeast_b200.h, "multi-discrete (factored) action spaces", states the rules).  An int `num_actions` is
the flat policy, unchanged.

UPGO, kickstarting and legal-action masks take flat rows only; a learner with a factored space raises for them before
anything is launched (check_learner).

Continuous action spaces: a net built with `num_actions=Gaussian(D)` has a diagonal-Gaussian policy over real vectors of
D dimensions, 1 <= D <= 64.  Its policy rows are [T, B, 2D], the mean mu in columns [0, D) and the log standard
deviation in [D, 2D), and its actions (and `last_action`) are float32 [T, B, D]: the unclipped samples, which an actor
clips to its environment's bounds itself before stepping it (include/torchbeast_b200.h, "continuous (diagonal-Gaussian)
action spaces", states the rules).  Such a net has num_actions = 2D and continuous_dim = D.  UPGO, kickstarting,
legal-action masks and integer actions are not built for it; check_learner raises for them.
"""
import ctypes
import dataclasses

import torch

from torchbeast_b200 import _lib

MAX_COMPONENTS = 16  # TB_MAX_ACTION_COMPONENTS
MAX_CONTINUOUS_DIM = 64  # TB_MAX_CONTINUOUS_DIM


@dataclasses.dataclass(frozen=True)
class Gaussian:
    """A continuous action space of `dim` real dimensions with a diagonal-Gaussian policy; pass it as a net's
    num_actions.  1 <= dim <= 64."""
    dim: int

    def __post_init__(self):
        if isinstance(self.dim, bool) or not isinstance(self.dim, int) or not 1 <= self.dim <= MAX_CONTINUOUS_DIM:
            raise _lib.TorchBeastB200Error("Gaussian(D) takes an int D in [1, %d], got %r"
                                           % (MAX_CONTINUOUS_DIM, self.dim))


class CActionSpace(ctypes.Structure):
    """tb_action_space, the host struct every factored entry point takes."""
    _fields_ = [("num_components", ctypes.c_int32), ("dims", ctypes.c_int32 * MAX_COMPONENTS)]


def dims_of(num_actions):
    """The component sizes (A_1, ..., A_D) of a tuple or list `num_actions`, checked (1 <= D <= 16, every A_k an int
    >= 1); None for an int (a flat policy) or a Gaussian (no discrete components)."""
    if isinstance(num_actions, (tuple, list)):
        dims = tuple(num_actions)
        if not 1 <= len(dims) <= MAX_COMPONENTS or any(
                isinstance(a, bool) or not isinstance(a, int) or a < 1 for a in dims):
            raise _lib.TorchBeastB200Error("a factored num_actions must be a tuple of 1 to %d ints >= 1, got %r"
                                           % (MAX_COMPONENTS, num_actions))
        return dims
    return None


def continuous_dim_of(num_actions):
    """D of a Gaussian(D) `num_actions`; None for an int or a tuple."""
    return num_actions.dim if isinstance(num_actions, Gaussian) else None


def width(num_actions):
    """The policy-logit width: num_actions itself, the sum of a tuple's component sizes, or 2D for a Gaussian(D)."""
    if isinstance(num_actions, Gaussian):
        return 2 * num_actions.dim
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
    """A model's component sizes, or None for a flat or a continuous policy."""
    return getattr(model, "action_dims", None)


def continuous_dim_of_model(model):
    """D of a model with a continuous (Gaussian) action space, or None."""
    return getattr(model, "continuous_dim", None)


def space_of_model(model):
    """A model's action space as its constructor took it: Gaussian(D), a tuple of component sizes, or the int width."""
    D = continuous_dim_of_model(model)
    if D is not None:
        return Gaussian(D)
    return dims_of_model(model) or model.num_actions


def loss_space_of_model(model):
    """The `action_space` argument of the loss wrappers for a model: Gaussian(D), its component sizes, or None."""
    D = continuous_dim_of_model(model)
    return Gaussian(D) if D is not None else dims_of_model(model)


def gaussian_mean(logits, D):
    """The eval-mode action of a Gaussian policy: the mean mu, float32 [T, B, D]."""
    return logits.detach()[..., :D].contiguous()


def gaussian_normal(logits, D):
    """torch.normal on (mu, exp(log sigma)), float32 [T, B, D]: what a continuous net samples without an
    ActionSampler."""
    logits = logits.detach()
    return torch.normal(logits[..., :D], logits[..., D:].exp())


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
    D = continuous_dim_of_model(model)
    if teacher is not None and (dims_of_model(teacher.net) != dims or continuous_dim_of_model(teacher.net) != D):
        raise _lib.TorchBeastB200Error("the teacher's action space %r differs from the learner's %r"
                                       % (space_of_model(teacher.net), space_of_model(model)))
    if D is not None:
        _check_continuous_learner(D, flags, batch)
        return
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


def _check_continuous_learner(D, flags, batch):
    """check_learner for a model with a Gaussian(D) space: UPGO, kickstarting, a legal_actions leaf and integer actions
    are not built for it."""
    not_built = []
    if getattr(flags, "upgo_cost", None) is not None:
        not_built.append("UPGO (flags.upgo_cost)")
    if getattr(flags, "kickstart_cost", None) is not None:
        not_built.append("kickstarting (flags.kickstart_cost)")
    if isinstance(batch, dict) and batch.get("legal_actions") is not None:
        not_built.append("legal-action masks (a legal_actions leaf)")
    if isinstance(batch, dict):
        for key in ("action", "last_action"):
            leaf = batch.get(key)
            if isinstance(leaf, torch.Tensor) and not leaf.dtype.is_floating_point:
                not_built.append("%s actions (%s %s; a continuous space takes float32 [T+1, B, %d])"
                                 % (leaf.dtype, key, tuple(leaf.shape), D))
    if not_built:
        raise _lib.TorchBeastB200Error("%s: not built for a continuous action space Gaussian(%d)"
                                       % (", ".join(not_built), D))
