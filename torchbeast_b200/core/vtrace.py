"""V-trace off-policy actor-critic targets - CUDA drop-in for torchbeast/core/vtrace.py.

Same names, signatures, return types and error text as the reference
(/root/reference/torchbeast/core/vtrace.py:36-139); every function launches hand-written
sm_90a kernels through the C-ABI (torchbeast_b200/csrc/vtrace.cu).  CUDA tensors only.
"""
import collections

import torch

from torchbeast_b200 import _lib

VTraceFromLogitsReturns = collections.namedtuple(
    "VTraceFromLogitsReturns",
    ["vs", "pg_advantages", "log_rhos", "behavior_action_log_probs", "target_action_log_probs"],
)

VTraceReturns = collections.namedtuple("VTraceReturns", "vs pg_advantages")

_SUFFIX = {torch.float32: "f32", torch.float64: "f64"}


def _suffix(t):
    try:
        return _SUFFIX[t.dtype]
    except KeyError:
        raise _lib.TorchBeastB200Error("torchbeast_b200: unsupported dtype %s (float32/float64 only)" % t.dtype)


class _ActionLogProbs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, policy_logits, actions):
        _lib.require_cuda(policy_logits, actions)
        A = policy_logits.shape[-1]
        logits2d = policy_logits.reshape(-1, A).contiguous()
        acts = actions.reshape(-1).to(torch.int64).contiguous()
        out = torch.empty(acts.shape, dtype=policy_logits.dtype, device=policy_logits.device)
        fn = getattr(_lib.lib(), "tb_action_log_probs_" + _suffix(policy_logits))
        _lib.check(fn(_lib.ptr(logits2d), _lib.ptr(acts), logits2d.shape[0], A, _lib.ptr(out), _lib.stream_ptr()),
                   "tb_action_log_probs")
        ctx.save_for_backward(logits2d, acts)
        ctx.logits_shape = policy_logits.shape
        return out.view_as(actions)

    @staticmethod
    def backward(ctx, grad_out):
        # d log pi(a) / d logits = onehot(a) - softmax(logits); off the learner's hot path
        # (learn() gets its gradients from the fused loss kernel).
        logits2d, acts = ctx.saved_tensors
        g = -torch.softmax(logits2d, dim=-1)
        g.scatter_add_(1, acts.unsqueeze(1), torch.ones_like(acts, dtype=g.dtype).unsqueeze(1))
        g = g * grad_out.reshape(-1, 1)
        return g.view(ctx.logits_shape), None


def action_log_probs(policy_logits, actions):
    """log pi(a|x) of the taken actions; reference vtrace.py:50-55."""
    return _ActionLogProbs.apply(policy_logits, actions)


@torch.no_grad()
def from_importance_weights(
    log_rhos,
    discounts,
    rewards,
    values,
    bootstrap_value,
    clip_rho_threshold=1.0,
    clip_pg_rho_threshold=1.0,
):
    """V-trace from log importance weights; reference vtrace.py:91-139 (one kernel launch)."""
    _lib.require_cuda(log_rhos, discounts, rewards, values, bootstrap_value)
    if bootstrap_value.dim() + 1 != values.dim():
        # The reference surfaces torch.cat's complaint (vtrace.py:111-113; vtrace_test.py:257-260).
        raise RuntimeError(
            "Tensors must have same number of dimensions: got %d and %d" % (values.dim(), bootstrap_value.dim() + 1))
    dtype = values.dtype
    sfx = _suffix(values)
    # Trailing dims broadcast like the reference (vtrace_test.py:229-241): flatten them into B.
    full = torch.broadcast_shapes(log_rhos.shape, discounts.shape, rewards.shape, values.shape,
                                  (1,) + tuple(bootstrap_value.shape))
    T = full[0]
    cols = 1
    for d in full[1:]:
        cols *= d

    def flat(x):
        return x.to(dtype).expand(full).reshape(T, cols).contiguous()

    lr, dc, rw, va = flat(log_rhos), flat(discounts), flat(rewards), flat(values)
    bs = bootstrap_value.to(dtype).expand(full[1:]).reshape(cols).contiguous()
    vs = torch.empty((T, cols), dtype=dtype, device=values.device)
    pg = torch.empty_like(vs)
    fn = getattr(_lib.lib(), "tb_vtrace_from_importance_weights_" + sfx)
    _lib.check(
        fn(_lib.ptr(lr), _lib.ptr(dc), _lib.ptr(rw), _lib.ptr(va), _lib.ptr(bs), T, cols,
           _lib.clip_arg(clip_rho_threshold), _lib.clip_arg(clip_pg_rho_threshold),
           _lib.ptr(vs), _lib.ptr(pg), _lib.stream_ptr()),
        "tb_vtrace_from_importance_weights")
    return VTraceReturns(vs=vs.view(full), pg_advantages=pg.view(full))


def _fused_from_logits(blogits, tlogits, actions, discounts, rewards, values, bootstrap, clip_rho, clip_pg):
    """One launch of the fused kernel (forward only): log-softmax picks, log-rho, scan."""
    T, B, A = tlogits.shape
    dev = values.device
    outs = [torch.empty((T, B), dtype=torch.float32, device=dev) for _ in range(5)]
    losses = torch.empty(4, dtype=torch.float32, device=dev)
    _lib.check(
        _lib.lib().tb_impala_loss_fwd_bwd_f32(
            _lib.ptr(blogits), _lib.ptr(tlogits), _lib.ptr(actions), _lib.ptr(rewards), None, _lib.ptr(discounts),
            _lib.ptr(values), _lib.ptr(bootstrap), T, B, A, 0.0, 0.0, 0.0, 0,
            _lib.clip_arg(clip_rho), _lib.clip_arg(clip_pg),
            *[_lib.ptr(o) for o in outs], _lib.ptr(losses), None, None, 0,
            _lib.ptr(_lib.workspace()), _lib.stream_ptr()),
        "tb_impala_loss_fwd_bwd_f32")
    vs, pg, lr, blp, tlp = outs
    return VTraceFromLogitsReturns(vs, pg, lr, blp, tlp)


def from_logits(
    behavior_policy_logits,
    target_policy_logits,
    actions,
    discounts,
    rewards,
    values,
    bootstrap_value,
    clip_rho_threshold=1.0,
    clip_pg_rho_threshold=1.0,
):
    """V-trace for softmax policies; reference vtrace.py:58-88.

    float32 [T,B,A] logits that do not require grad take the single fused launch; anything
    else (float64, extra dims, logits that need d(log pi)/d(logits)) is composed from
    action_log_probs + from_importance_weights exactly like the reference."""
    tensors = (behavior_policy_logits, target_policy_logits, actions, discounts, rewards, values, bootstrap_value)
    _lib.require_cuda(*tensors)
    plain = (
        target_policy_logits.dim() == 3 and values.dim() == 2 and bootstrap_value.dim() == 1
        and all(t.dtype == torch.float32 for t in tensors if t is not actions)
        and behavior_policy_logits.shape == target_policy_logits.shape
        and discounts.shape == values.shape == rewards.shape == actions.shape == target_policy_logits.shape[:2]
        and not (torch.is_grad_enabled() and (behavior_policy_logits.requires_grad or target_policy_logits.requires_grad))
    )
    if plain:
        return _fused_from_logits(
            behavior_policy_logits.contiguous(), target_policy_logits.contiguous(),
            actions.to(torch.int64).contiguous(), discounts.contiguous(), rewards.contiguous(),
            values.detach().contiguous(), bootstrap_value.detach().contiguous(),
            clip_rho_threshold, clip_pg_rho_threshold)
    tlp = action_log_probs(target_policy_logits, actions)
    blp = action_log_probs(behavior_policy_logits, actions)
    log_rhos = tlp - blp
    vs, pg = from_importance_weights(
        log_rhos, discounts, rewards, values, bootstrap_value, clip_rho_threshold, clip_pg_rho_threshold)
    return VTraceFromLogitsReturns(vs, pg, log_rhos, blp, tlp)
