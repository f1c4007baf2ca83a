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
import torch

from torchbeast_b200 import _lib


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

    def sample(self, logits, stream_ids=None):
        """logits: [T, B, A] float32 CUDA tensor -> int64 [T, B] actions; advances `step` by T.

        Row (t, b) uses counter step + t and stream id `stream_ids[b]` (int64 [B], any device; default: the column
        index b).  A row containing NaN, with every logit -inf, or with a +inf logit gets action -1."""
        _lib.require_cuda(logits)
        if logits.dim() != 3 or logits.dtype != torch.float32:
            raise _lib.TorchBeastB200Error("logits must be float32 [T, B, A], got %s %r" % (logits.dtype, tuple(logits.shape)))
        T, B, A = logits.shape
        logits = logits.detach().contiguous()
        if stream_ids is not None:
            if tuple(stream_ids.shape) != (B,):
                raise _lib.TorchBeastB200Error("stream_ids must have shape [B] = [%d], got %r" % (B, tuple(stream_ids.shape)))
            stream_ids = stream_ids.to(device=logits.device, dtype=torch.int64).contiguous()
        actions = torch.empty(T, B, dtype=torch.int64, device=logits.device)
        _lib.check(
            _lib.lib().tb_sample_actions_f32(_lib.ptr(logits), T, B, A, self.seed % 2 ** 64, self.step % 2 ** 64,
                                             _lib.ptr(stream_ids), _lib.ptr(actions), _lib.stream_ptr()),
            "tb_sample_actions_f32")
        self.step += T
        return actions

    def __repr__(self):
        return "ActionSampler(seed=%d, step=%d)" % (self.seed, self.step)
