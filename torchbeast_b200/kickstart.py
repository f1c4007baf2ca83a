"""Kickstarting (Schmitt et al. 2018, "Kickstarting Deep Reinforcement Learning", arXiv:1803.03835): distil a frozen
teacher policy into the learner inside the learn step.

    model.teacher = Teacher(teacher_net)      # any net of this package, at any precision
    flags.kickstart_cost = 1.0                # None or absent: off; anneal it to 0 between steps

With a cost, learn() runs `teacher_net.learner_forward` on the step's batch (the mixed one with replay) right after the
learner's forward, and one more launch after the loss (tb_kickstart_loss_f32) adds
kickstart_cost * sum_{t,b} w_b KL(pi_teacher,t || pi_learner,t) to the total loss and its gradient
kickstart_cost * w_b * (pi_learner - pi_teacher) to the policy logits' gradient (w_b: the prioritised-replay weight of
column b, or 1).  The stats gain kickstart_loss and teacher_kl (sum KL / (T*B), unweighted).

An LSTM teacher starts every unroll from its zero state and resets on `done` as usual: the batch carries no teacher
state.  A feed-forward teacher is exact.  A zero cost leaves the learner's update bit for bit, but the teacher forward
still runs: detach the teacher (model.teacher = None) once the cost reaches 0.

Teacher is a plain class, not an nn.Module, so attaching it does not add the teacher's keys to the learner's
state_dict: the learner's checkpoints stay the reference's, and the teacher is not saved with them."""
import numbers

import torch

from torchbeast_b200 import _lib


def kickstart_cost(flags):
    """flags.kickstart_cost as a finite float >= 0, or None when the flag is None or absent (no kickstarting).  Raises
    ValueError for a negative, NaN, infinite, boolean or non-numeric value, before anything is launched."""
    v = getattr(flags, "kickstart_cost", None)
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, numbers.Real):
        raise ValueError("kickstart_cost must be None or a finite number >= 0, got %r" % (v,))
    cost = float(v)
    if not 0.0 <= cost < float("inf"):  # NaN fails too
        raise ValueError("kickstart_cost must be finite and >= 0 (or None), got %r" % (v,))
    return cost


_BARE_NET = ("model.teacher is a %s, an nn.Module: torch registers it as a submodule, so its keys would enter the "
             "learner's state_dict; attach it as model.teacher = torchbeast_b200.kickstart.Teacher(net)")


def teacher_of(model):
    """model.teacher (a Teacher) or None.  Raises when it is an nn.Module or anything else but a Teacher."""
    t = getattr(model, "teacher", None)
    if t is None or isinstance(t, Teacher):
        return t
    if isinstance(t, torch.nn.Module):
        raise _lib.TorchBeastB200Error(_BARE_NET % type(t).__name__)
    raise _lib.TorchBeastB200Error("model.teacher must be a torchbeast_b200.kickstart.Teacher or None, got %s"
                                   % type(t).__name__)


def _flat_range(net):
    flat = net.flat_params
    return flat.data_ptr(), flat.data_ptr() + flat.numel() * flat.element_size()


class Teacher:
    """A frozen teacher network for kickstarting (see the module docstring).  `net` is any network of this package
    (AtariNet or ResNet, any precision, with or without LSTM or num_tasks: only its policy logits are read).  Its
    weights are never written by learn(); load new ones in place with teacher.net.load_state_dict(...), which a
    graphed learner follows on its next replay."""

    def __init__(self, net):
        if not all(hasattr(net, a) for a in ("learner_forward", "flat_params", "num_actions", "observation_shape")):
            raise _lib.TorchBeastB200Error("Teacher needs a torchbeast_b200 network (AtariNet or ResNet), got %s"
                                           % type(net).__name__)
        self.net = net
        self._zero = {}

    def initial_state(self, batch_size):
        """The zero LSTM state of width `batch_size` every unroll starts from, kept per width so that a captured step
        allocates nothing; () for a feed-forward teacher."""
        key = (int(batch_size), self.net.flat_params.device)
        state = self._zero.get(key)
        if state is None:
            state = self._zero[key] = tuple(self.net.initial_state(int(batch_size)))
        return state

    def check(self, model, actor_model=None):
        """Raises unless the teacher can run beside `model`: on its device, with its num_actions and
        observation_shape, and neither `model` nor `actor_model` nor sharing their flat parameter buffers (its forward
        would overwrite the learner's saved activations, or race with the acting threads)."""
        net = self.net
        if net.flat_params.device != model.flat_params.device:
            raise _lib.TorchBeastB200Error("the teacher is on %s, the learner on %s"
                                           % (net.flat_params.device, model.flat_params.device))
        if net.num_actions != model.num_actions:
            raise _lib.TorchBeastB200Error("the teacher has num_actions %d, the learner %d"
                                           % (net.num_actions, model.num_actions))
        t_obs, m_obs = tuple(net.observation_shape), tuple(getattr(model, "observation_shape", ()))
        if t_obs != m_obs:
            raise _lib.TorchBeastB200Error("the teacher's observation_shape %r is not the learner's %r" % (t_obs, m_obs))
        lo, hi = _flat_range(net)
        for name, other in (("learner model", model), ("actor model", actor_model)):
            if other is None:
                continue
            if other is net:
                raise _lib.TorchBeastB200Error("the teacher's net is the %s; give it a network of its own" % name)
            olo, ohi = _flat_range(other)
            if lo < ohi and olo < hi:
                raise _lib.TorchBeastB200Error("the teacher's net shares the %s's flat parameter buffer" % name)

    def logits(self, batch):
        """The teacher's policy logits [T+1, B, A] on `batch` (learner_forward from the zero state)."""
        return self.net.learner_forward(batch, self.initial_state(batch["reward"].shape[1])).policy_logits
