"""Seeded, reproducible action sampling for the acting forward (tb_sample_actions_f32, csrc/sample.cu).

The reference samples with `torch.multinomial(F.softmax(policy_logits, dim=1), num_samples=1)` (monobeast.py:618-619,
polybeast_learner.py:256-257), which draws from torch's global generator: an action then depends on everything else that
consumed that generator and on how rows happened to be batched.  Here an action depends only on (seed, step, stream id,
logits row), so the same seed replays an actor's actions.

Attach a sampler to a network to use it in training-mode forwards (the eval path stays greedy):

    model.action_sampler = ActionSampler(seed=1234)

The forward then passes `inputs["stream_ids"]` (int64 [B]) to the sampler when the inputs carry it, and otherwise
uses each row's batch column as its stream id.
"""
import ctypes

import torch

from torchbeast_b200 import _lib, action_space


class ActionSampler:
    """Counter-based categorical sampler.  `seed` and `step` are plain public ints, so a checkpoint can store them and
    a restored sampler continues the same sequence.

    Each `sample` call reads `step` on the host and passes it to the kernel by value, then advances it by T.  The call
    itself is therefore not CUDA-graph safe: a captured launch would replay the same step forever.  To replay the acting
    forward as a graph, use torchbeast_b200.acting.GraphedActor: it captures tb_sample_actions_dev_f32, which reads
    (seed, step) from device memory, publishes this sampler's `seed` and `step` there before each replay and advances
    `step` as an eager call does, so graphed and eager calls give one action sequence.  Calls from several threads
    must be serialised by the caller (polybeast_learner.inference already holds its lock around the forward)."""

    def __init__(self, seed, step=0):
        self.seed = int(seed)
        self.step = int(step)

    def sample(self, logits, stream_ids=None, action_dims=None, continuous_dim=None):
        """logits: [T, B, A] float32 CUDA tensor -> int64 [T, B] actions; advances `step` by T.

        Row (t, b) uses counter step + t and stream id `stream_ids[b]` (int64 [B], any device; default: the column
        index b).  A row containing NaN, with every logit -inf, or with a +inf logit gets action -1.

        action_dims (A_1, ..., A_D), summing to A: a factored policy (torchbeast_b200.action_space), sampled by
        tb_sample_actions_factored_f32 into int64 [T, B, D]; component k draws from its own segment of the row, and a
        segment with no distribution gets -1.

        continuous_dim D, with A = 2D: a Gaussian policy (torchbeast_b200.action_space.Gaussian), sampled by
        tb_sample_gaussian_f32 into float32 [T, B, D]; a component with a non-finite mean or log-std gets NaN."""
        _lib.require_cuda(logits)
        if logits.dim() != 3 or logits.dtype != torch.float32:
            raise _lib.TorchBeastB200Error("logits must be float32 [T, B, A], got %s %r" % (logits.dtype, tuple(logits.shape)))
        T, B, A = logits.shape
        logits = logits.detach().contiguous()
        if stream_ids is not None:
            if tuple(stream_ids.shape) != (B,):
                raise _lib.TorchBeastB200Error("stream_ids must have shape [B] = [%d], got %r" % (B, tuple(stream_ids.shape)))
            stream_ids = stream_ids.to(device=logits.device, dtype=torch.int64).contiguous()
        if action_dims is not None:
            actions = sample_factored(logits, action_dims, stream_ids, seed=self.seed, step=self.step)
            self.step += T
            return actions
        if continuous_dim is not None:
            actions = sample_gaussian(logits, continuous_dim, stream_ids, seed=self.seed, step=self.step)
            self.step += T
            return actions
        actions = torch.empty(T, B, dtype=torch.int64, device=logits.device)
        _lib.check(
            _lib.lib().tb_sample_actions_f32(_lib.ptr(logits), T, B, A, self.seed % 2 ** 64, self.step % 2 ** 64,
                                             _lib.ptr(stream_ids), _lib.ptr(actions), _lib.stream_ptr()),
            "tb_sample_actions_f32")
        self.step += T
        return actions

    def __repr__(self):
        return "ActionSampler(seed=%d, step=%d)" % (self.seed, self.step)


def sample_factored(logits, action_dims, stream_ids=None, seed=0, step=0, seed_step=None):
    """tb_sample_actions_factored_f32 on contiguous float32 logits [T, B, sum(action_dims)] -> int64 [T, B, D].  The
    (seed, step) it samples at is `seed_step` (int64 [2] on the device, read when the kernel runs: graph-capturable)
    when given, else the host ints `seed` and `step`.  stream_ids: int64 [B] on the logits' device, or None."""
    T, B, A = logits.shape
    dims = action_space.dims_of(tuple(action_dims))
    actions = torch.empty(T, B, len(dims), dtype=torch.int64, device=logits.device)
    _lib.check(
        _lib.lib().tb_sample_actions_factored_f32(
            _lib.ptr(logits), T, B, A, seed % 2 ** 64, step % 2 ** 64, _lib.ptr(seed_step), _lib.ptr(stream_ids),
            ctypes.byref(action_space.c_space(dims)), _lib.ptr(actions), _lib.stream_ptr()),
        "tb_sample_actions_factored_f32")
    return actions


def sample_gaussian(logits, continuous_dim, stream_ids=None, seed=0, step=0, seed_step=None):
    """tb_sample_gaussian_f32 on contiguous float32 rows [T, B, 2D] (mu, log sigma) -> float32 [T, B, D], D =
    continuous_dim.  (seed, step) and stream_ids as in sample_factored."""
    T, B, A = logits.shape
    if A != 2 * int(continuous_dim):
        raise _lib.TorchBeastB200Error("a Gaussian(%d) policy takes rows [T, B, %d], got %r"
                                       % (continuous_dim, 2 * int(continuous_dim), tuple(logits.shape)))
    actions = torch.empty(T, B, int(continuous_dim), dtype=torch.float32, device=logits.device)
    _lib.check(
        _lib.lib().tb_sample_gaussian_f32(
            _lib.ptr(logits), T, B, A, seed % 2 ** 64, step % 2 ** 64, _lib.ptr(seed_step), _lib.ptr(stream_ids),
            _lib.ptr(actions), _lib.stream_ptr()),
        "tb_sample_gaussian_f32")
    return actions
