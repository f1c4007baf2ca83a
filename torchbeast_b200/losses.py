"""The three IMPALA loss terms as CUDA autograd functions.

Mirror of compute_baseline_loss / compute_entropy_loss / compute_policy_gradient_loss
(/root/reference/torchbeast/monobeast.py:107-125 == polybeast_learner.py:113-131): same
names, sum reduction, float32 or float64 inputs, advantages receive no gradient.  Each
forward is one launch that also emits the closed-form gradient (SURVEY.md 8(a) A4); the
backward only scales it by the incoming scalar.  learn() does not use these - it calls the
fully fused kernel (tb_impala_loss_f32) - they exist for API parity.
"""
import torch

from torchbeast_b200 import _lib
from torchbeast_b200.core.vtrace import _suffix


class _BaselineLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, advantages):
        _lib.require_cuda(advantages)
        adv = advantages.contiguous()
        out = torch.empty(1, dtype=adv.dtype, device=adv.device)
        grad = torch.empty_like(adv) if advantages.requires_grad else None
        fn = getattr(_lib.lib(), "tb_baseline_loss_" + _suffix(adv))
        _lib.check(fn(_lib.ptr(adv), adv.numel(), _lib.ptr(out), _lib.ptr(grad), _lib.ptr(_lib.workspace()),
                      _lib.stream_ptr()), "tb_baseline_loss")
        ctx.grad = grad
        return out[0]

    @staticmethod
    def backward(ctx, g):
        return ctx.grad * g


class _EntropyLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits):
        _lib.require_cuda(logits)
        A = logits.shape[-1]
        x = logits.reshape(-1, A).contiguous()
        out = torch.empty(1, dtype=x.dtype, device=x.device)
        grad = torch.empty_like(x) if logits.requires_grad else None
        fn = getattr(_lib.lib(), "tb_entropy_loss_" + _suffix(x))
        _lib.check(fn(_lib.ptr(x), x.shape[0], A, _lib.ptr(out), _lib.ptr(grad), _lib.ptr(_lib.workspace()),
                      _lib.stream_ptr()), "tb_entropy_loss")
        ctx.grad, ctx.shape = grad, logits.shape
        return out[0]

    @staticmethod
    def backward(ctx, g):
        return (ctx.grad * g).view(ctx.shape)


class _PolicyGradientLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, actions, advantages):
        _lib.require_cuda(logits, actions, advantages)
        A = logits.shape[-1]
        x = logits.reshape(-1, A).contiguous()
        a = actions.reshape(-1).to(torch.int64).contiguous()
        adv = advantages.detach().reshape(-1).to(x.dtype).contiguous()
        out = torch.empty(1, dtype=x.dtype, device=x.device)
        grad = torch.empty_like(x) if logits.requires_grad else None
        fn = getattr(_lib.lib(), "tb_pg_loss_" + _suffix(x))
        _lib.check(fn(_lib.ptr(x), _lib.ptr(a), _lib.ptr(adv), x.shape[0], A, _lib.ptr(out), _lib.ptr(grad),
                      _lib.ptr(_lib.workspace()), _lib.stream_ptr()), "tb_pg_loss")
        ctx.grad, ctx.shape = grad, logits.shape
        return out[0]

    @staticmethod
    def backward(ctx, g):
        return (ctx.grad * g).view(ctx.shape), None, None


def compute_baseline_loss(advantages):
    return _BaselineLoss.apply(advantages)


def compute_entropy_loss(logits):
    """Return the entropy loss, i.e., the negative entropy of the policy."""
    return _EntropyLoss.apply(logits)


def compute_policy_gradient_loss(logits, actions, advantages):
    return _PolicyGradientLoss.apply(logits, actions, advantages)
