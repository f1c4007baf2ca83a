"""Legal-action masks ("invalid action masking": AlphaStar, OpenAI Five; Huang & Ontañón, "A Closer Look at Invalid
Action Masking in Policy Gradient Algorithms", FLAIRS 2022): sample, act greedily and learn over each step's legal
actions.

A rollout or acting input may carry a leaf legal_actions bool / uint8 [T+1, B, A] (acting: [1, B, A]), nonzero =
legal, indexed like `frame`: row t holds the actions legal at frame t.  In monobeast's act() loop it is an env output,
stored at row t+1 beside frame t+1, while behaviour logits row t+1 and action row t+1 were formed at frame t.  So:

  * a net's forward output row t is masked by legal_actions row t (AtariNet / ResNet do it themselves, see mask_policy);
  * the behaviour logits policy_logits[1:] are masked by legal_actions[:-1] (learn_step, one launch);
  * action[1:] is checked against legal_actions[:-1], on the behaviour copy and on the learner's rows [:-1] (one more
    launch): an illegal taken action makes the step's losses NaN.

An illegal logit becomes MASKED_LOGIT = torch.finfo(torch.float32).min, finite on purpose: every kernel downstream then
computes the softmax over the legal set with p = 0 and a gradient of +-0 at an illegal entry (include/torchbeast_b200.h,
tb_mask_logits_f32).  A row with no legal action is left unmasked."""
import torch

from torchbeast_b200 import _lib

MASKED_LOGIT = torch.finfo(torch.float32).min
LEAF = "legal_actions"


def _legal_bytes(legal, shape):
    """`legal` as contiguous uint8 bytes after checking it is bool or uint8 of `shape` on a CUDA device."""
    _lib.require_cuda(legal)
    if legal.dtype not in (torch.bool, torch.uint8) or tuple(legal.shape) != tuple(shape):
        raise _lib.TorchBeastB200Error("legal_actions must be bool or uint8 %r, got %s %r"
                                       % (tuple(shape), legal.dtype, tuple(legal.shape)))
    return legal.contiguous().view(torch.uint8)


@torch.no_grad()
def mask_logits(logits, legal, actions=None, fill=MASKED_LOGIT, out=None):
    """One tb_mask_logits_f32 launch over float32 logits [..., A] and legal [..., A] (bool or uint8, nonzero = legal):
    on every row with a legal entry, out = legal ? logits : fill; a row with none is copied.  `actions` (integer
    [...], optional): a row whose in-range action is illegal becomes NaN.  `out`: a contiguous float32 tensor of
    logits' shape (it may be `logits` itself, when contiguous: in place), or None for a new one.  Returns out."""
    _lib.require_cuda(logits)
    if logits.dtype != torch.float32 or logits.dim() < 1:
        raise _lib.TorchBeastB200Error("logits must be float32 [..., A], got %s %r" % (logits.dtype, tuple(logits.shape)))
    A = logits.shape[-1]
    lb = _legal_bytes(legal, logits.shape)
    x = logits.contiguous()
    if out is None:
        out = torch.empty_like(x)
    elif out.dtype != torch.float32 or tuple(out.shape) != tuple(logits.shape) or not out.is_contiguous() \
            or out.device != logits.device:
        raise _lib.TorchBeastB200Error("out must be a contiguous float32 %r on %s" % (tuple(logits.shape), logits.device))
    if actions is not None:
        _lib.require_cuda(actions)
        if tuple(actions.shape) != tuple(logits.shape[:-1]):
            raise _lib.TorchBeastB200Error("actions must be %r, got %r" % (tuple(logits.shape[:-1]), tuple(actions.shape)))
        actions = actions.to(torch.int64).contiguous()
    p = _lib.ptr
    _lib.check(_lib.lib().tb_mask_logits_f32(p(x), p(out), p(lb), p(actions), x.numel() // A if A else 0, A, float(fill),
                                             _lib.stream_ptr()),
               "tb_mask_logits_f32")
    return out


class _MaskLogits(torch.autograd.Function):
    """The masked logits of a net's autograd forward: the mask out of place with the sentinel, and its gradient
    (legal ? g : 0 on a masked row, g on a row with no legal action) by the same kernel with fill = 0."""

    @staticmethod
    def forward(ctx, logits, legal):
        ctx.legal = legal
        return mask_logits(logits.detach(), legal)

    @staticmethod
    def backward(ctx, g):
        return mask_logits(g.contiguous(), ctx.legal, fill=0.0), None


def mask_policy(logits, inputs):
    """A net's policy logits [T, B, A] masked by inputs["legal_actions"] (no leaf: `logits` as they are).  The leaf must
    be bool or uint8 [T, B, A] on the logits' device.  Under autograd (logits that require grad) the mask is a
    _MaskLogits node; otherwise it runs in place."""
    legal = inputs.get(LEAF) if isinstance(inputs, dict) else None
    if legal is None:
        return logits
    if legal.device != logits.device:
        raise _lib.TorchBeastB200Error("legal_actions is on %s, the net on %s" % (legal.device, logits.device))
    if logits.requires_grad and torch.is_grad_enabled():
        _legal_bytes(legal, logits.shape)
        return _MaskLogits.apply(logits, legal)
    return mask_logits(logits, legal, out=logits)


def check_leaf(batch):
    """Raises TorchBeastB200Error unless batch["legal_actions"], when present, is bool or uint8 (T+1, B, A) with the
    shape and device of batch["policy_logits"].  Runs before anything is staged or launched."""
    legal = batch.get(LEAF) if isinstance(batch, dict) else None
    if legal is None:
        return
    logits = batch.get("policy_logits")
    if logits is None:
        raise _lib.TorchBeastB200Error("a batch with legal_actions needs policy_logits [T+1, B, A]")
    if legal.dtype not in (torch.bool, torch.uint8) or tuple(legal.shape) != tuple(logits.shape):
        raise _lib.TorchBeastB200Error("legal_actions must be bool or uint8 (T+1, B, A) = %r like policy_logits, got %s %r"
                                       % (tuple(logits.shape), legal.dtype, tuple(legal.shape)))
    if legal.device != logits.device:
        raise _lib.TorchBeastB200Error("legal_actions is on %s, policy_logits on %s" % (legal.device, logits.device))
