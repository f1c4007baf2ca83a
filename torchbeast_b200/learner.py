"""Fused pieces of the learner step shared by monobeast.learn and polybeast_learner.learn."""
import collections
import ctypes
import numbers
import os
import threading

import numpy as np
import torch

from torchbeast_b200 import _lib
from torchbeast_b200 import action_space as _action_space
from torchbeast_b200.kickstart import kickstart_cost, teacher_of
from torchbeast_b200.legal_actions import LEAF as _LEGAL, check_leaf as _check_legal, mask_logits

ImpalaLoss = collections.namedtuple(
    "ImpalaLoss",
    "vs pg_advantages log_rhos behavior_action_log_probs target_action_log_probs losses grad_logits grad_values",
)
# What the trust-region loss returns next to its ImpalaLoss: kl float32 [T, B] = KL(pi_t || mu_t) of every row, sums
# float32 [2] = {number of trusted rows, sum of kl over all rows}.
TrustRegion = collections.namedtuple("TrustRegion", "kl sums")
# What the loss returns last when given upgo_cost: adv float32 [T, B] = the UPGO advantage of every row, loss float32
# [1] = upgo_cost * sum w_b * (-log pi(a)) * adv (already included in losses[3]).
Upgo = collections.namedtuple("Upgo", "adv loss")
# What kickstart_loss returns: loss float32 [1] = cost * sum w_b * KL_t (already included in losses[3]), kl_sum float32
# [1] = sum KL_t over all T*B rows, unweighted.
Kickstart = collections.namedtuple("Kickstart", "loss kl_sum")

# tb_hparams (include/torchbeast_b200.h): the loss and optimizer values the entry points read from device memory.
# tb_hparams_layout() reports the compiled layout; tests/test_graph_hparams_cpu.py checks this record against it.
HPARAMS = np.dtype([
    ("beta1", "<f8"), ("beta2", "<f8"), ("discounting", "<f4"), ("baseline_cost", "<f4"), ("entropy_cost", "<f4"),
    ("clip_rho", "<f4"), ("clip_pg_rho", "<f4"), ("clip_rewards", "<i4"), ("max_norm", "<f4"), ("alpha", "<f4"),
    ("eps", "<f4"), ("momentum", "<f4"), ("weight_decay", "<f4")], align=True)


def _clip_rewards(reward_clipping):
    if reward_clipping not in ("abs_one", "none"):
        raise ValueError("reward_clipping must be 'abs_one' or 'none'")
    return int(reward_clipping == "abs_one")


def pack_hparams(flags, optimizer=None, clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0):
    """The tb_hparams record of one learn() step, as a 0-dim NumPy array of HPARAMS: the loss values and the gradient
    clip from `flags`, the optimizer's from `optimizer.param_groups[0]` (a FusedOptimizer; fields it does not use stay
    0).  Raises what the eager step would raise for the same values, so nothing is captured or replayed with them."""
    rec = np.zeros((), HPARAMS)
    rec["discounting"] = flags.discounting
    rec["baseline_cost"] = flags.baseline_cost
    rec["entropy_cost"] = flags.entropy_cost
    rec["clip_rewards"] = _clip_rewards(flags.reward_clipping)
    rec["clip_rho"] = _lib.clip_arg(clip_rho_threshold)
    rec["clip_pg_rho"] = _lib.clip_arg(clip_pg_rho_threshold)
    rec["max_norm"] = -1.0 if flags.grad_norm_clipping is None else float(flags.grad_norm_clipping)
    if optimizer is not None:
        for k, v in optimizer.hparams().items():
            rec[k] = v
    return rec


def publish_hparams(rec, block):
    """Enqueue the copy of record `rec` into the device block `block` (uint8 [HPARAMS.itemsize]) on the current stream.
    The source is a fresh pinned buffer: the caching host allocator does not hand it out again until the copy is done."""
    host = torch.empty(HPARAMS.itemsize, dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = np.frombuffer(rec.tobytes(), dtype=np.uint8)
    block.copy_(host, non_blocking=True)


def trust_region_kl(flags):
    """flags.trust_region_kl as a float beta >= 0 (+inf allowed), or None when the flag is None or absent (no trust
    region).  Raises ValueError for a negative, NaN or non-numeric value, before anything is launched."""
    v = getattr(flags, "trust_region_kl", None)
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, numbers.Real):
        raise ValueError("trust_region_kl must be None or a number >= 0, got %r" % (v,))
    beta = float(v)
    if not beta >= 0.0:  # NaN fails too
        raise ValueError("trust_region_kl must be >= 0 (or None), got %r" % (v,))
    return beta


def upgo_cost(flags):
    """flags.upgo_cost as a finite float >= 0, or None when the flag is None or absent (no UPGO).  Raises ValueError for
    a negative, NaN, infinite, boolean or non-numeric value, before anything is launched."""
    v = getattr(flags, "upgo_cost", None)
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, numbers.Real):
        raise ValueError("upgo_cost must be None or a finite number >= 0, got %r" % (v,))
    cost = float(v)
    if not 0.0 <= cost < float("inf"):  # NaN fails too
        raise ValueError("upgo_cost must be finite and >= 0 (or None), got %r" % (v,))
    return cost


def _device_scalar(value, name, device, finite=False):
    """The device float32 [1] a kernel reads when it runs: `value` itself when it is a tensor (a graph's published
    scalar), else a new one holding float(value), which must be >= 0 (and finite with `finite`)."""
    if isinstance(value, torch.Tensor):
        _lib.require_cuda(value)
        if value.dtype != torch.float32 or value.numel() != 1:
            raise _lib.TorchBeastB200Error("%s must be a float or a float32 device scalar, got %s %r" % (
                name, value.dtype, tuple(value.shape)))
        return value
    x = float(value)
    if not (0.0 <= x < float("inf") if finite else x >= 0.0):
        raise ValueError("%s must be >= 0%s, got %r" % (name, " and finite" if finite else "", value))
    return torch.full((1,), x, dtype=torch.float32, device=device)


def hparams_field(block, name):
    """Field `name` of a device tb_hparams block as a 0-dim tensor view (float32 / float64 / int32)."""
    dt, off = HPARAMS.fields[name]
    torch_dtype = {"<f4": torch.float32, "<f8": torch.float64, "<i4": torch.int32}[dt.str]
    return block[off:off + dt.itemsize].view(torch_dtype).view(())


@torch.no_grad()
def impala_loss_fwd_bwd(
    behavior_policy_logits,
    target_policy_logits,
    actions,
    rewards,
    done,
    values,
    bootstrap_value,
    discounting=0.99,
    baseline_cost=0.5,
    entropy_cost=0.0006,
    reward_clipping="abs_one",
    clip_rho_threshold=1.0,
    clip_pg_rho_threshold=1.0,
    with_grads=True,
    hparams_dev=None,
    column_weights=None,
    trust_region=None,
    upgo_cost=None,
    action_space=None,
):
    """The whole loss block of learn() in ONE kernel launch (tb_impala_loss_f32), two with UPGO.

    Inputs are the shifted [T,B,...] slices (batch[1:], learner_outputs[:-1]); `done` is a
    bool/uint8 tensor.  Replaces monobeast.py:245-277 / polybeast_learner.py:332-361 and the
    autograd graph behind them: returns vs / pg_advantages / log-rhos, losses =
    [pg, baseline_cost*baseline, entropy_cost*entropy, total] and d total / d(target logits,
    values) laid out as [T+1,B,...] with a zero bootstrap row, ready for the network backward.

    With `hparams_dev` (a device tb_hparams block, see pack_hparams / publish_hparams) the kernel reads discounting,
    the costs, the reward clip and the two V-trace clips from the block when it runs, and the corresponding arguments
    are not used: a captured CUDA graph then follows what is published between replays.

    With `column_weights` (float32 [B], device) the pg, baseline and entropy terms of column b, in the losses and the
    gradients, are multiplied by column_weights[b] (prioritised replay's importance weights); weights of 1.0 give the
    unweighted bits.

    With `trust_region` (beta: a float >= 0, or a float32 device scalar read when the kernel runs) a row whose
    KL(pi || mu) exceeds beta gets rho = 0 in the V-trace and the policy gradient (the rule is stated with
    tb_impala_loss_f32 in include/torchbeast_b200.h), and the call returns (ImpalaLoss, TrustRegion).  vs and
    pg_advantages are the masked ones; log_rhos and the log-probabilities are not masked.

    With `upgo_cost` (a finite float >= 0, or a float32 device scalar read when the kernel runs) the upgoing policy
    gradient (tb_upgo_loss_f32, a second launch; the rule is stated in include/torchbeast_b200.h) adds
    upgo_cost * sum w_b * (-log pi(a)) * A_upgo to losses[3] and its gradient to grad_logits, and an Upgo(adv, loss)
    is appended last to what the call returns.

    With `action_space` (component sizes (A_1, ..., A_D) summing to A; torchbeast_b200.action_space) the policy is
    factored: `actions` are int64 [T, B, D] and tb_impala_loss_factored_f32 forms every row quantity per component
    (the rules are stated in include/torchbeast_b200.h).  UPGO takes flat rows only.

    With `action_space` a Gaussian(D) (torchbeast_b200.action_space) the policy is a diagonal Gaussian: the logits are
    the (mu, log sigma) rows [T, B, 2D], `actions` are float32 [T, B, D] and tb_impala_loss_gaussian_f32 forms the
    log-densities, the entropy, the trust region's KL and the gradients (the rules are stated in
    include/torchbeast_b200.h).  UPGO takes categorical rows only.
    """
    tensors = (behavior_policy_logits, target_policy_logits, actions, rewards, done, values, bootstrap_value)
    _lib.require_cuda(*tensors)
    if column_weights is not None:
        _lib.require_cuda(column_weights)
        if column_weights.dtype != torch.float32 or column_weights.numel() != target_policy_logits.shape[1]:
            raise _lib.TorchBeastB200Error("column_weights must be float32 [%d], got %s %r" % (
                target_policy_logits.shape[1], column_weights.dtype, tuple(column_weights.shape)))
    loss, _, trust, upgo = _impala_loss(
        behavior_policy_logits, target_policy_logits, actions, rewards, done, values, bootstrap_value, discounting,
        baseline_cost, entropy_cost, reward_clipping, clip_rho_threshold, clip_pg_rho_threshold, with_grads,
        hparams_dev, column_weights=column_weights, trust_region=trust_region, upgo_cost=upgo_cost,
        action_space=action_space)
    out = (loss,) + tuple(x for x in (trust, upgo) if x is not None)
    return out[0] if len(out) == 1 else out


@torch.no_grad()
def impala_loss_popart(
    behavior_policy_logits,
    target_policy_logits,
    actions,
    rewards,
    done,
    values,
    task,
    mu,
    nu,
    discounting=0.99,
    baseline_cost=0.5,
    entropy_cost=0.0006,
    reward_clipping="abs_one",
    clip_rho_threshold=1.0,
    clip_pg_rho_threshold=1.0,
    hparams_dev=None,
    trust_region=None,
    upgo_cost=None,
    action_space=None,
):
    """impala_loss_fwd_bwd on a PopArt-normalised value head (tb_impala_loss_f32 with a task).

    `values` is the normalised head output n [T+1, B, K] with its bootstrap row, `task` int64 [T+1, B] the task of each
    of those rows, `mu` / `nu` float64 [K] the statistics.  The V-trace runs on sigma_k * n[k] + mu_k; vs and
    pg_advantages are unnormalised, the losses and gradients are taken in normalised space, and grad_values is
    [T+1, B, K].  A row with a task id outside [0, K) adds no loss and gets zero gradient rows.  Returns
    (ImpalaLoss, task_sums): task_sums float64 [3, K] = per-task count, sum vs, sum vs^2 over rows t < T, the input
    of popart_update (SUM all-reduce it first when data-parallel).  With `trust_region` (see impala_loss_fwd_bwd) it
    returns (ImpalaLoss, task_sums, TrustRegion), task_sums from the masked vs.  With `upgo_cost` (see
    impala_loss_fwd_bwd; its advantage is divided by sigma_k) an Upgo is appended last.  `action_space`: a factored
    or a Gaussian policy, as in impala_loss_fwd_bwd."""
    tensors = (behavior_policy_logits, target_policy_logits, actions, rewards, done, values, task, mu, nu)
    _lib.require_cuda(*tensors)
    T, B, A = target_policy_logits.shape
    K = values.shape[-1]
    if tuple(values.shape) != (T + 1, B, K) or tuple(task.shape) != (T + 1, B):
        raise _lib.TorchBeastB200Error("PopArt values must be [T+1, B, K] and task [T+1, B] for T, B = %d, %d; got %r, %r"
                                       % (T, B, tuple(values.shape), tuple(task.shape)))
    if mu.dtype != torch.float64 or nu.dtype != torch.float64 or mu.numel() != K or nu.numel() != K:
        raise _lib.TorchBeastB200Error("PopArt mu / nu must be float64 [%d]" % K)
    loss, sums, trust, upgo = _impala_loss(
        behavior_policy_logits, target_policy_logits, actions, rewards, done, values, None, discounting,
        baseline_cost, entropy_cost, reward_clipping, clip_rho_threshold, clip_pg_rho_threshold, True, hparams_dev,
        popart=(task, mu, nu), trust_region=trust_region, upgo_cost=upgo_cost, action_space=action_space)
    return (loss, sums) + tuple(x for x in (trust, upgo) if x is not None)


def _impala_loss(behavior_policy_logits, target_policy_logits, actions, rewards, done, values, bootstrap_value,
                 discounting, baseline_cost, entropy_cost, reward_clipping, clip_rho_threshold, clip_pg_rho_threshold,
                 with_grads, hparams_dev, column_weights=None, popart=None, trust_region=None, upgo_cost=None,
                 action_space=None):
    """The tb_impala_loss_f32 call behind impala_loss_fwd_bwd and impala_loss_popart, on inputs they checked, and with
    `upgo_cost` the tb_upgo_loss_f32 call right behind it on the same inputs.  popart: None, or (task, mu, nu) with
    values [T+1, B, K].  action_space: component sizes, for tb_impala_loss_factored_f32, or a Gaussian(D), for
    tb_impala_loss_gaussian_f32.  Returns (ImpalaLoss, task_sums or None, TrustRegion or None, Upgo or None)."""
    D = _action_space.continuous_dim_of(action_space)
    dims = None if D is not None else _action_space.dims_of(None if action_space is None else tuple(action_space))
    if D is not None:
        if upgo_cost is not None:
            raise _lib.TorchBeastB200Error("UPGO (upgo_cost) is not built for a continuous action space Gaussian(%d)" % D)
        T, B, A = target_policy_logits.shape
        if A != 2 * D or tuple(actions.shape) != (T, B, D) or not actions.dtype.is_floating_point:
            raise _lib.TorchBeastB200Error(
                "a continuous action space Gaussian(%d) takes logits [T, B, 2D] and float actions [T, B, D] = %r, got "
                "logits %r and %s actions %r" % (D, (T, B, D), tuple(target_policy_logits.shape), actions.dtype,
                                                 tuple(actions.shape)))
    if dims is not None:
        if upgo_cost is not None:
            raise _lib.TorchBeastB200Error("UPGO (upgo_cost) is not built for a factored action space %r" % (dims,))
        T, B = target_policy_logits.shape[:2]
        if tuple(actions.shape) != (T, B, len(dims)):
            raise _lib.TorchBeastB200Error("a factored action space %r takes actions [T, B, D] = %r, got %r"
                                           % (dims, (T, B, len(dims)), tuple(actions.shape)))
    if hparams_dev is None:
        clip_rewards = _clip_rewards(reward_clipping)
    else:
        _lib.require_cuda(hparams_dev)
        discounting = hparams_field(hparams_dev, "discounting")  # uint8 done: the discounts below read the block
        clip_rewards = 0
    T, B, A = target_policy_logits.shape
    dev = values.device
    f32 = torch.float32
    if done.dtype == torch.bool:
        dn, disc = done.contiguous().view(torch.uint8), None
    elif done.dtype == torch.uint8:
        # `~done` on uint8 is a bitwise NOT in the reference (SURVEY Appendix A): discount = (255-done)*gamma
        dn, disc = None, ((~done).to(f32) * discounting).contiguous()
    else:
        raise _lib.TorchBeastB200Error("done must be bool or uint8")
    task = mu = nu = sums = bs = None
    K = 0
    if popart is not None:
        task, mu, nu = popart
        K = values.shape[-1]
        task, mu, nu = task.to(torch.int64).contiguous(), mu.contiguous(), nu.contiguous()
        sums = torch.empty((3, K), dtype=torch.float64, device=dev)
    else:
        bs = bootstrap_value.detach().to(f32).contiguous()
    beta = kl = kl_sums = None
    if trust_region is not None:
        beta = _device_scalar(trust_region, "trust_region", dev)
        kl, kl_sums = torch.empty((T, B), dtype=f32, device=dev), torch.empty(2, dtype=f32, device=dev)
    cost = None if upgo_cost is None else _device_scalar(upgo_cost, "upgo_cost", dev, finite=True)
    cw = None if column_weights is None else column_weights.contiguous()
    outs = [torch.empty((T, B), dtype=f32, device=dev) for _ in range(5)]
    losses = torch.empty(4, dtype=f32, device=dev)
    gl = torch.empty((T + 1, B, A), dtype=f32, device=dev) if with_grads else None
    gv = torch.empty((T + 1, B) + ((K,) if popart is not None else ()), dtype=f32, device=dev) if with_grads else None
    tl = target_policy_logits.detach().to(f32).contiguous()
    act = actions.to(torch.int64 if D is None else f32).contiguous()
    rw, vals = rewards.to(f32).contiguous(), values.detach().to(f32).contiguous()
    disc_arg = 0.0 if hparams_dev is not None else float(discounting)
    p = _lib.ptr
    ws = _lib.workspace()
    args = (p(behavior_policy_logits.to(f32).contiguous()), p(tl), p(act), p(rw), p(dn), p(disc), p(vals), p(bs),
            T, B, A, disc_arg, float(baseline_cost), float(entropy_cost),
            clip_rewards, _lib.clip_arg(clip_rho_threshold), _lib.clip_arg(clip_pg_rho_threshold), p(hparams_dev),
            p(cw), p(task), p(mu), p(nu), K, p(sums), p(beta), p(kl), p(kl_sums),
            *[p(o) for o in outs], p(losses), p(gl), p(gv), 1)
    if D is not None:
        _lib.check(_lib.lib().tb_impala_loss_gaussian_f32(*args, p(ws), _lib.stream_ptr()), "tb_impala_loss_gaussian_f32")
    elif dims is None:
        _lib.check(_lib.lib().tb_impala_loss_f32(*args, p(ws), _lib.stream_ptr()), "tb_impala_loss_f32")
    else:
        _lib.check(_lib.lib().tb_impala_loss_factored_f32(*args, ctypes.byref(_action_space.c_space(dims)), p(ws),
                                                          _lib.stream_ptr()),
                   "tb_impala_loss_factored_f32")
    upgo = None
    if cost is not None:
        upgo = Upgo(torch.empty((T, B), dtype=f32, device=dev), torch.empty(1, dtype=f32, device=dev))
        _lib.check(
            _lib.lib().tb_upgo_loss_f32(
                p(tl), p(act), p(rw), p(dn), p(disc), p(vals), p(bs), T, B, A, disc_arg, clip_rewards,
                _lib.clip_arg(clip_pg_rho_threshold), p(hparams_dev), p(cw), p(task), p(mu), p(nu), K, p(outs[2]),
                p(beta), p(kl), p(cost), p(upgo.adv), p(upgo.loss), p(losses), p(gl), p(ws), _lib.stream_ptr()),
            "tb_upgo_loss_f32")
    return ImpalaLoss(*outs, losses, gl, gv), sums, None if beta is None else TrustRegion(kl, kl_sums), upgo


@torch.no_grad()
def kickstart_loss(teacher_logits, target_logits, losses, grad_logits, cost, column_weights=None):
    """The kickstarting term (tb_kickstart_loss_f32, one launch; the rule is stated in include/torchbeast_b200.h):
    cost * sum_{t,b} w_b KL(p_teacher,t || p_learner,t) over the [T, B, A] logits (the [:-1] rows of the two forward
    outputs), ADDED into `losses[3]` (float32 [4], the loss's) and, unless `grad_logits` is None, its gradient
    cost * w_b * (p_learner - p_teacher) ADDED into rows t < T of `grad_logits` (float32 [T or T+1, B, A]).  A zero
    cost writes neither.  `cost`: a finite float >= 0, or a float32 device scalar read when the kernel runs.
    `column_weights`: float32 [B] (w_b), or None for 1.  Returns Kickstart(loss, kl_sum)."""
    _lib.require_cuda(teacher_logits, target_logits, losses)
    T, B, A = target_logits.shape
    f32 = torch.float32
    if tuple(teacher_logits.shape) != (T, B, A):
        raise _lib.TorchBeastB200Error("teacher logits %r do not match the learner's %r"
                                       % (tuple(teacher_logits.shape), (T, B, A)))
    if losses.dtype != f32 or losses.numel() != 4 or not losses.is_contiguous():
        raise _lib.TorchBeastB200Error("losses must be contiguous float32 [4], got %s %r"
                                       % (losses.dtype, tuple(losses.shape)))
    if grad_logits is not None:
        _lib.require_cuda(grad_logits)
        if grad_logits.dtype != f32 or not grad_logits.is_contiguous() or tuple(grad_logits.shape) not in (
                (T, B, A), (T + 1, B, A)):
            raise _lib.TorchBeastB200Error("grad_logits must be contiguous float32 [T(+1), B, A] for %r, got %s %r"
                                           % ((T, B, A), grad_logits.dtype, tuple(grad_logits.shape)))
    if column_weights is not None:
        _lib.require_cuda(column_weights)
        if column_weights.dtype != f32 or column_weights.numel() != B:
            raise _lib.TorchBeastB200Error("column_weights must be float32 [%d], got %s %r" % (
                B, column_weights.dtype, tuple(column_weights.shape)))
        column_weights = column_weights.contiguous()
    dev = target_logits.device
    c = _device_scalar(cost, "kickstart_cost", dev, finite=True)
    out = torch.empty(2, dtype=f32, device=dev)
    p = _lib.ptr
    _lib.check(
        _lib.lib().tb_kickstart_loss_f32(
            p(teacher_logits.detach().to(f32).contiguous()), p(target_logits.detach().to(f32).contiguous()), T, B, A,
            p(column_weights), p(c), p(out), p(losses), p(grad_logits), p(_lib.workspace()), _lib.stream_ptr()),
        "tb_kickstart_loss_f32")
    return Kickstart(out[:1], out[1:])


@torch.no_grad()
def popart_update(task_sums, beta, mu, nu, weight, bias):
    """PopArt statistics update and output-preserving value-head rescale, in place (tb_popart_update): `beta` is a
    float64 device scalar, `weight` [K, F] / `bias` [K] the value head (views of the flat parameter buffer)."""
    _lib.require_cuda(task_sums, beta, mu, nu, weight, bias)
    K, F = weight.shape
    for t, dt in ((task_sums, torch.float64), (beta, torch.float64), (mu, torch.float64), (nu, torch.float64),
                  (weight, torch.float32), (bias, torch.float32)):
        if t.dtype != dt or not t.is_contiguous():
            raise _lib.TorchBeastB200Error("popart_update: expected contiguous %s, got %s" % (dt, t.dtype))
    if task_sums.numel() != 3 * K or mu.numel() != K or nu.numel() != K or bias.numel() != K or beta.numel() != 1:
        raise _lib.TorchBeastB200Error("popart_update: sizes disagree with weight [%d, %d]" % (K, F))
    p = _lib.ptr
    _lib.check(_lib.lib().tb_popart_update(p(task_sums), p(beta), p(mu), p(nu), K, p(weight), p(bias), F,
                                           _lib.stream_ptr()),
               "tb_popart_update")


def _popart_task(model, batch):
    """batch["task"] as int64 [T+1, B]; optional (all zeros) for a single-task model."""
    task = batch.get("task")
    if task is None:
        if model.popart.num_tasks > 1:
            raise _lib.TorchBeastB200Error("a model with num_tasks > 1 needs batch['task']")
        return torch.zeros(batch["reward"].shape[:2], dtype=torch.int64, device=batch["reward"].device)
    return task.to(torch.int64)


def _dp_world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size()
    return 1


def _all_reduce_grads(flat_grad):
    """Batch-column data parallelism (SURVEY.md 8(e)): losses are sums over (t, b), so one
    SUM all-reduce of the flat gradient over NCCL/NVLink reproduces the single-GPU gradient;
    every rank then clips and steps on the reduced gradient and replicas stay identical."""
    import torch.distributed as dist

    if _dp_world() > 1:
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM)
        return True
    return False


_ar_streams = {}


def _backward_with_overlapped_all_reduce(model, grad_logits, grad_values):
    """Network backward + the gradient SUM all-reduce, still one logical SUM per parameter, in two buckets in reverse
    forward order (SURVEY 8(e) G1): the LSTM + heads slice (17 of 24 MB; final after backward phase 1) is reduced on a
    side stream WHILE the conv/fc trunk backward runs, the trunk slice right after it.  Fork / join are events, so the
    whole thing is captured into the learner's CUDA graph.  Falls back to one all-reduce after the backward when the
    model has no two-phase backward."""
    import torch.distributed as dist
    if _dp_world() <= 1:
        return model.learner_backward(grad_logits, grad_values)
    if not hasattr(model, "grad_split") or os.environ.get("TB_AR_OVERLAP", "1") == "0":
        fg = model.learner_backward(grad_logits, grad_values)
        dist.all_reduce(fg, op=dist.ReduceOp.SUM)
        return fg
    dev = model.flat_params.device
    on_gpu = dev.type == "cuda"   # (the gloo / CPU path of tests/test_dist_cpu.py runs the same bucket logic without streams)
    side = main = None
    if on_gpu:
        side = _ar_streams.get(dev)
        if side is None:
            side = _ar_streams[dev] = torch.cuda.Stream(device=dev)
        main = torch.cuda.current_stream(dev)
    state = {"split": 0}

    def between(fg, split):
        state["split"] = split
        if split > 0:
            if on_gpu:
                side.wait_stream(main)        # phase 1 (heads + LSTM gradients) is enqueued on main
                with torch.cuda.stream(side):
                    dist.all_reduce(fg[split:], op=dist.ReduceOp.SUM)
            else:
                dist.all_reduce(fg[split:], op=dist.ReduceOp.SUM)

    fg = model.learner_backward(grad_logits, grad_values, between=between, **({"aux_stream": side} if on_gpu else {}))
    split = state["split"]
    if split > 0:
        dist.all_reduce(fg[:split], op=dist.ReduceOp.SUM)
        if on_gpu:
            main.wait_stream(side)
    else:
        dist.all_reduce(fg, op=dist.ReduceOp.SUM)
    return fg


def optimizer_step(model, optimizer, max_grad_norm, hparams_dev=None):
    from torchbeast_b200 import optim as _optim

    if isinstance(optimizer, _optim.FusedOptimizer):
        # fused clip + update on the flat buffers, 2-3 launches
        optimizer.step(max_grad_norm=max_grad_norm, hparams_dev=hparams_dev)
    else:
        # foreign optimizer object: gradients are already in .grad (views of the flat buffer)
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)
        optimizer.step()


DEFAULT_POPART_BETA = 3e-4


def popart_beta(flags):
    return float(getattr(flags, "popart_beta", DEFAULT_POPART_BETA))


def _popart_stats(mu, nu):
    """The stats-dict entries of a PopArt model from host copies of its statistics."""
    sigma = [float(min(max(max(n - m * m, 0.0) ** 0.5, 1e-4), 1e6)) for m, n in zip(mu.tolist(), nu.tolist())]
    return {"popart_mu": mu.tolist(), "popart_sigma": sigma}


_POPART_PRIORITIZED = ("prioritised replay does not support PopArt (model.popart): weighted per-task statistics and "
                       "normalised priorities are not defined; use a uniform ReplayBuffer (no priority_exponent)")


def _check_replay(model):
    replay = getattr(model, "replay", None)
    if replay is not None and replay.prioritized and getattr(model, "popart", None) is not None:
        raise _lib.TorchBeastB200Error(_POPART_PRIORITIZED)


def learn_step(flags, model, actor_model, batch, initial_agent_state, optimizer, scheduler,
               behavior_logits=None, actions=None, stats_sync=True, hparams_dev=None, popart_beta_dev=None,
               fresh_columns=None, draw=None, trust_beta_dev=None, upgo_cost_dev=None, kickstart_cost_dev=None):
    """One optimisation step on a [T+1, B, ...] rollout batch (dict of CUDA tensors).

    Launch sequence (no autograd graph, no host sync until the stats read-back):
      network forward -> fused V-trace + 3 losses + their gradients (1 launch) -> network
      backward into the flat gradient -> [NCCL all-reduce] -> fused clip + optimizer step -> actor copy.
    With `hparams_dev` (GraphedLearner's device tb_hparams block) the loss and the optimizer read the values of
    `flags` and of the optimizer's param group from the block, not from the host.

    A model built with `num_tasks` (PopArt, model.popart) runs the PopArt loss instead (impala_loss_popart, one more
    launch for the per-task sums), SUM all-reduces the sums when data-parallel, and after the optimizer step updates the
    statistics and rescales the value head (popart_update) before the actor copy.  beta is `popart_beta_dev` (a float64
    device scalar, GraphedLearner's) or flags.popart_beta.

    `fresh_columns` (a replay-mixed batch, see torchbeast_b200.replay): the stats' episode returns come from columns
    [0, fresh_columns) only, so a replayed episode end is not counted twice; the losses cover the whole batch.

    A model with running observation statistics (an MLPNet built with normalize_observations=True, model.obs_norm)
    merges rows 1..T of the fresh columns [0, fresh_columns) of batch["frame"] into them after the optimizer step (two
    launches; the sums SUM all-reduced when data-parallel), before the actor copy, which takes the new statistics.  The
    step's own forward normalised with the statistics as they were before it.

    `draw` (a prioritised buffer's replay.Draw, or one built by hand): with `draw.weights` the loss is the importance-
    weighted one (impala_loss_fwd_bwd with column_weights), so the stats' loss values are the weighted sums; with
    `draw.buffer` its priorities are updated from the loss's vs and values at `draw.slots`, right after the loss.

    flags.trust_region_kl (a float beta >= 0; None or absent: off) runs the trust-region loss: rows with
    KL(pi || mu) > beta get rho = 0 in the V-trace and the policy gradient, on every column, fresh and replayed.  beta
    is `trust_beta_dev` (a float32 device scalar, GraphedLearner's) or the flag.  The stats then carry
    trust_fraction (trusted rows / T*B) and mean_policy_kl (sum KL / T*B), read back with the loss values; a prioritised
    buffer's priorities come from the masked vs.

    flags.upgo_cost (a finite float >= 0; None or absent: off) adds the upgoing policy gradient (tb_upgo_loss_f32, one
    more launch right after the loss) on every path above.  The cost is `upgo_cost_dev` (a float32 device scalar,
    GraphedLearner's) or the flag.  The stats then carry upgo_loss, which total_loss includes.

    flags.kickstart_cost (a finite float >= 0; None or absent: off) distils the teacher attached as model.teacher (a
    torchbeast_b200.kickstart.Teacher) into the learner on every path above: the teacher's forward runs on the same
    batch right after the learner's, and kickstart_loss (one launch after the loss and UPGO) adds its term to the total
    and to grad_logits.  The cost is `kickstart_cost_dev` (a float32 device scalar, GraphedLearner's) or the flag.  The
    stats then carry kickstart_loss, which total_loss includes, and teacher_kl (sum KL / T*B, unweighted).

    A model with a factored action space (model.action_dims, torchbeast_b200.action_space) takes action [T+1, B, D] and
    runs the factored loss (tb_impala_loss_factored_f32) on every path above but UPGO and kickstarting.

    A model with a continuous action space (model.continuous_dim, a Gaussian(D)) takes float32 action [T+1, B, D] and
    policy_logits [T+1, B, 2D] and runs the Gaussian loss (tb_impala_loss_gaussian_f32) on every path above but UPGO,
    kickstarting and legal-action masks.

    A batch with a legal_actions leaf (bool or uint8 [T+1, B, A], torchbeast_b200.legal_actions) learns over each
    step's legal actions on every path above: the learner's and the teacher's forwards mask their own logits, and one
    launch writes a masked copy of the behaviour logits (policy_logits[1:] or `behavior_logits`) under
    legal_actions[:-1], checking action[1:] against it; one more checks it in place on the learner's rows [:-1] (an
    illegal taken action makes the losses NaN).  The loss, the trust region, UPGO and kickstarting read that copy.
    """
    pop = getattr(model, "popart", None)
    if draw is not None and pop is not None:
        raise _lib.TorchBeastB200Error(_POPART_PRIORITIZED)
    beta = trust_region_kl(flags)
    trust_region = None if beta is None else (beta if trust_beta_dev is None else trust_beta_dev)
    cost = upgo_cost(flags)
    upgo_arg = None if cost is None else (cost if upgo_cost_dev is None else upgo_cost_dev)
    ks_cost = kickstart_cost(flags)
    teacher = _teacher_for(model, actor_model, ks_cost)
    ks_arg = None if ks_cost is None else (ks_cost if kickstart_cost_dev is None else kickstart_cost_dev)
    trust = upgo = ks = None
    out = model.learner_forward(batch, initial_agent_state)
    teacher_logits = None if teacher is None else teacher.logits(batch)
    blogits = (batch["policy_logits"] if behavior_logits is None else behavior_logits)[1:]
    acts = batch["action"] if actions is None else actions
    legal = batch.get(_LEGAL)
    if legal is not None:
        # the behaviour logits row t+1 and action row t+1 were formed at frame t, whose legal set is row t
        blogits = mask_logits(blogits.detach().to(torch.float32), legal[:-1], actions=acts[1:])
        # the same check on the learner's own rows (already masked by its forward, so only a NaN row can change): a NaN
        # behaviour row alone would not reach the losses, as the rho clips (fminf) drop a NaN log-rho
        mask_logits(out.policy_logits[:-1], legal[:-1], actions=acts[1:], out=out.policy_logits[:-1])
    if pop is None:
        loss = impala_loss_fwd_bwd(
            blogits, out.policy_logits[:-1], acts[1:], batch["reward"][1:], batch["done"][1:],
            out.baseline[:-1], out.baseline[-1],
            discounting=flags.discounting, baseline_cost=flags.baseline_cost, entropy_cost=flags.entropy_cost,
            reward_clipping=flags.reward_clipping, hparams_dev=hparams_dev,
            column_weights=None if draw is None else draw.weights, trust_region=trust_region, upgo_cost=upgo_arg,
            action_space=_action_space.loss_space_of_model(model))
        if trust_region is not None or upgo_arg is not None:
            loss, *rest = loss
            trust = rest.pop(0) if trust_region is not None else None
            upgo = rest.pop(0) if upgo_arg is not None else None
        grad_values = loss.grad_values
        if draw is not None and draw.buffer is not None:
            draw.buffer.update_priorities(loss.vs, out.baseline[:-1], draw.slots)
    else:
        values = out.baseline.reshape(out.baseline.shape[:2] + (pop.num_tasks,))
        res = impala_loss_popart(
            blogits, out.policy_logits[:-1], acts[1:], batch["reward"][1:], batch["done"][1:], values,
            _popart_task(model, batch), pop.mu, pop.nu,
            discounting=flags.discounting, baseline_cost=flags.baseline_cost, entropy_cost=flags.entropy_cost,
            reward_clipping=flags.reward_clipping, hparams_dev=hparams_dev, trust_region=trust_region,
            upgo_cost=upgo_arg, action_space=_action_space.loss_space_of_model(model))
        loss, task_sums, *rest = res
        trust = rest.pop(0) if trust_region is not None else None
        upgo = rest.pop(0) if upgo_arg is not None else None
        grad_values = loss.grad_values.view(out.baseline.shape)
    if teacher is not None:
        ks = kickstart_loss(teacher_logits[:-1], out.policy_logits[:-1], loss.losses, loss.grad_logits, ks_arg,
                            column_weights=None if draw is None else draw.weights)
    _backward_with_overlapped_all_reduce(model, loss.grad_logits, grad_values)
    optimizer_step(model, optimizer, flags.grad_norm_clipping, hparams_dev=hparams_dev)
    if pop is not None:
        if _dp_world() > 1:
            import torch.distributed as dist
            dist.all_reduce(task_sums, op=dist.ReduceOp.SUM)  # every rank applies the global batch's update
        if popart_beta_dev is None:
            popart_beta_dev = torch.full((1,), popart_beta(flags), dtype=torch.float64, device=task_sums.device)
        weight, bias = model.value_head()
        popart_update(task_sums, popart_beta_dev, pop.mu, pop.nu, weight, bias)
    if getattr(model, "obs_norm", None) is not None:
        obs_sums = model.obs_norm_sums(batch["frame"], fresh_columns)
        if _dp_world() > 1:
            import torch.distributed as dist
            dist.all_reduce(obs_sums, op=dist.ReduceOp.SUM)  # every rank merges the global batch's rows
        model.obs_norm_update(obs_sums)
    if scheduler is not None:
        scheduler.step()
    if actor_model is not None and actor_model is not model:
        if hasattr(actor_model, "copy_params_from") and hasattr(model, "flat_params"):
            actor_model.copy_params_from(model)
        else:
            actor_model.load_state_dict(model.state_dict())
    if not stats_sync:
        return dict(losses=loss.losses, vtrace=loss, trust=trust, upgo=upgo, kickstart=ks)
    done, ep_ret = batch["done"][1:], batch["episode_return"][1:]
    if fresh_columns is not None:
        done, ep_ret = done[:, :fresh_columns], ep_ret[:, :fresh_columns]
    episode_returns = ep_ret[done.bool()]
    # the step's one blocking read-back: the loss values, and the trust-region sums, UPGO and kickstarting values behind
    # them
    host = _loss_values(loss.losses, trust, upgo, ks).cpu()
    ep = episode_returns.cpu()
    stats = {
        "episode_returns": tuple(ep.numpy()),
        "mean_episode_return": torch.mean(ep).item(),
        "total_loss": host[3].item(),
        "pg_loss": host[0].item(),
        "baseline_loss": host[1].item(),
        "entropy_loss": host[2].item(),
    }
    stats.update(_extra_stats(host, None if trust is None else trust.kl.numel(), upgo is not None,
                              _kickstart_rows(ks, loss)))
    if pop is not None:
        stats.update(_popart_stats(pop.mu.cpu(), pop.nu.cpu()))
    return stats


def _teacher_for(model, actor_model, cost):
    """The Teacher the step runs (model.teacher, checked against the learner), or None when kickstarting is off
    (`cost` None).  Raises before anything is launched: for a bare nn.Module as model.teacher whatever the cost, and
    for a cost without a teacher or a teacher that cannot run beside the learner (kickstart.Teacher.check)."""
    teacher = teacher_of(model)
    if cost is None:
        return None
    if teacher is None:
        raise _lib.TorchBeastB200Error("flags.kickstart_cost is set but the learner has no teacher: attach one as "
                                       "model.teacher = torchbeast_b200.kickstart.Teacher(net), or set the cost to None")
    teacher.check(model, actor_model)
    return teacher


def _kickstart_rows(ks, loss):
    """T*B, the rows teacher_kl averages over, or None without kickstarting."""
    return None if ks is None else loss.vs.numel()


def _loss_values(losses, trust, upgo, ks=None):
    """The device values the stats read back at once: losses [4], then the trust-region sums [2], the UPGO loss [1]
    and the kickstarting loss and KL sum [2] when they are on."""
    parts = [losses] + ([] if trust is None else [trust.sums]) + ([] if upgo is None else [upgo.loss]) + (
        [] if ks is None else [ks.loss, ks.kl_sum])
    return parts[0] if len(parts) == 1 else torch.cat(parts)


def _extra_stats(host, trust_rows, has_upgo, kickstart_rows=None):
    """The trust-region, UPGO and kickstarting stats entries from a host copy of _loss_values; trust_rows None: no
    trust region; kickstart_rows (T*B) None: no kickstarting."""
    stats = {}
    i = 4 if trust_rows is None else 6
    if has_upgo:
        stats["upgo_loss"] = host[i].item()
        i += 1
    if kickstart_rows is not None:
        stats["kickstart_loss"] = host[i].item()
        stats["teacher_kl"] = host[i + 1].item() / kickstart_rows
    if trust_rows is not None:
        stats.update(_trust_stats(host[4:6], trust_rows))
    return stats


def _trust_stats(sums, rows):
    """The stats-dict entries of the trust region from a host copy of its two sums over `rows` rows."""
    return {"trust_fraction": sums[0].item() / rows, "mean_policy_kl": sums[1].item() / rows}


def _graph_enabled(flags):
    """The graphed step is opt-in: flags.cuda_graph (or TB_CUDA_GRAPH=1).  Capture costs four throw-away steps and pins the
    batch shape; a training loop that calls learn() thousands of times with one shape wants it, a unit test does not."""
    import os
    v = getattr(flags, "cuda_graph", None)
    if v is None:
        v = os.environ.get("TB_CUDA_GRAPH", "0") not in ("0", "", "false")
    return bool(v)


def _is_host(batch):
    t = batch["frame"] if isinstance(batch, dict) else batch[0]
    return not t.is_cuda


def learn(flags, model, actor_model, batch, initial_agent_state, optimizer, scheduler, lock=None):
    """What monobeast.learn / polybeast_learner.learn run per rollout batch.

    * `batch` may live on the HOST (the reference's learner-queue nest / monobeast buffers): it is staged through the
      model's RolloutStager (pinned slot -> one async H2D copy on the copy stream) OUTSIDE `lock`, exactly where the
      reference does its `.to(device)` (polybeast_learner.py:307 - so with two learner threads the copy of one thread
      overlaps the other thread's step), then consumed under the lock.
    * with flags.cuda_graph (or TB_CUDA_GRAPH=1) the device side is ONE CUDA-graph replay (GraphedLearner, created on first
      use per batch shape); otherwise the eager launch sequence of learn_step.
    * with a replay buffer attached as `model.replay` (torchbeast_b200.replay.ReplayBuffer), the staged batch and state
      are mixed with replayed columns under the lock, inside the graph when graphed; the warm-up phase and the mixing
      phase are two graphs, as their batch widths differ.  A prioritised buffer adds its draw, the weighted loss and
      the priority update to the same sequence (learn_step's `draw`); with PopArt it raises.
    * a legal_actions leaf (torchbeast_b200.legal_actions) is checked first, then staged, graphed and replayed like
      any other leaf; learn_step learns over each step's legal actions.
    * a model with a factored action space (torchbeast_b200.action_space) learns on action [T+1, B, D] on every path
      above; UPGO, kickstarting, a legal_actions leaf or a teacher with another space raise before anything is staged.
    * a model with a continuous action space (Gaussian(D)) learns on float32 action [T+1, B, D] on every path above;
      UPGO, kickstarting, a legal_actions leaf, a teacher with another space or integer actions raise before anything
      is staged.
    * an MLPNet (float32 observation vectors) learns on a float32 frame leaf [T+1, B, O] on every path above; a
      frame_history, an unstacked or uint8 frame leaf or another O raise before anything is staged.  With
      normalize_observations its running statistics are updated after each step (learn_step), inside the graph too.
    * with flags.kickstart_cost, the teacher attached as model.teacher (torchbeast_b200.kickstart.Teacher) runs on the
      same (mixed) batch and its KL term joins the loss (learn_step); the teacher is part of the graph's structure.
    Returns the reference's stats dict."""
    import contextlib
    from torchbeast_b200 import staging
    # raises before anything is staged or launched: an invalid legal_actions leaf, an invalid cost, a cost without a
    # usable teacher, a bare net
    _check_legal(batch)
    teacher = _teacher_for(model, actor_model, kickstart_cost(flags))
    _action_space.check_learner(model, flags, batch, teacher_of(model))
    if hasattr(model, "check_batch"):  # MLPNet: a float32 [T+1, B, O] frame leaf
        model.check_batch(batch)
    needs_last_action = getattr(model, "needs_last_action", False) or (
        teacher is not None and getattr(teacher.net, "needs_last_action", False))
    slot = None
    stager = None
    if _is_host(batch):
        stager = getattr(model, "_tb_stager", None)
        if stager is None or not all(k in stager.spec and stager.spec[k] == (tuple(v.shape), v.dtype) for k, v in batch.items()):
            stager = staging.RolloutStager(staging.spec_like(batch), model.flat_params.device, depth=3)
            model._tb_stager = stager
        slot = stager.put(batch)
        initial_agent_state = tuple(t.to(model.flat_params.device, non_blocking=True) for t in initial_agent_state)
    snap = None
    with (lock if lock is not None else contextlib.nullcontext()):
        if stager is not None:
            # this thread's own slot: wait for ITS copy (slots complete in submission order per thread)
            torch.cuda.current_stream().wait_event(stager._ready[slot])
            with stager._lock:
                if slot in stager._submitted:
                    stager._submitted.remove(slot)
            batch = stager.dev[slot]
        if "last_action" not in batch and needs_last_action:
            # the polybeast nest has no separate last_action leaf: row t of `action` IS the action taken before frame t
            batch = dict(batch, last_action=batch["action"])
        try:
            _check_replay(model)
            if _graph_enabled(flags):
                _require_fused(optimizer)
                hparams = pack_hparams(flags, optimizer)  # raises before anything is captured or replayed
                structure = GraphedLearner.structure_of(optimizer, batch, flags, model)
                graphs = model.__dict__.setdefault("_tb_graphs", {})
                gkey = (tuple((k, tuple(v.shape)) for k, v in batch.items() if k in GraphedLearner.KEYS), id(optimizer),
                        id(actor_model))
                replay = getattr(model, "replay", None)
                if replay is not None:
                    gkey += (id(replay), replay.mixing(replay.prepare(batch, initial_agent_state)))
                gl = graphs.get(gkey)
                if gl is None or gl.structure != structure:
                    # a value that chooses a kernel or a buffer changed, so the eager step would switch too: replay the
                    # graph of the new structure, captured now or kept from before; the current one stays cached
                    if gl is not None:
                        graphs[gkey + (gl.structure,)] = gl
                    gl = graphs.pop(gkey + (structure,), None)
                    if gl is None:
                        gl = GraphedLearner(flags, model, actor_model, optimizer, batch, initial_agent_state)
                    graphs[gkey] = gl
                gl.step(batch, initial_agent_state, scheduler, hparams)
                if stager is not None:
                    stager.release(slot)  # the inputs now live in the graph's static buffers
                    slot = None
                if os.environ.get("TB_STATS_IN_LOCK", "0") == "1":   # the reference's behaviour: read back under the lock
                    return gl.stats()
                snap = gl.snapshot()      # tiny device copies, still under the lock (the next replay overwrites the originals)
                snap_event = torch.cuda.Event()
                snap_event.record()
            else:
                fresh = draw = None
                replay = getattr(model, "replay", None)
                if replay is not None:
                    batch, initial_agent_state, fresh = replay.mix(batch, initial_agent_state)
                    draw = replay.last_draw if replay.prioritized else None
                return learn_step(flags, model, actor_model, batch, initial_agent_state, optimizer, scheduler,
                                  fresh_columns=fresh, draw=draw)
        finally:
            if stager is not None and slot is not None:
                stager.release(slot)
    # graphed path: the blocking stats read-back happens OUTSIDE the lock - the device work of this step is already
    # enqueued, so another learner thread can enqueue its step right behind it (the reference holds its lock across the
    # .item() calls, polybeast_learner.py:373-379, which idles the GPU for a host round trip per step)
    return GraphedLearner.stats_from(snap, snap_event)


def shard_rollout(batch, initial_agent_state, rank, world_size):
    """Batch-column partition for data-parallel learners (SURVEY.md 8(e) G1): rank g of G takes
    columns [g*B/G, (g+1)*B/G) of every [T+1, B, ...] leaf and of the [layers, B, H] LSTM state.
    V-trace, the LSTM and the convs are per-column and the losses are sums, so the SUM all-reduce
    of the shards' gradients equals the full-batch gradient."""
    def cols(t, dim):
        B = t.shape[dim]
        if B % world_size:
            raise ValueError("batch size %d is not divisible by world size %d" % (B, world_size))
        n = B // world_size
        return t.narrow(dim, rank * n, n).contiguous()

    if isinstance(batch, dict):
        shard = {k: cols(v, 1) for k, v in batch.items()}
    else:
        shard = type(batch)(cols(v, 1) for v in batch)
    state = tuple(cols(s, 1) for s in initial_agent_state)
    return shard, state


def _require_fused(optimizer):
    from torchbeast_b200 import optim as _optim
    if not isinstance(optimizer, _optim.FusedOptimizer):
        raise _lib.TorchBeastB200Error(
            "GraphedLearner needs a fused optimizer from torchbeast_b200.optim (RMSprop, Adam or AdamW)")


class GraphedLearner:
    """The whole device side of learn() captured ONCE into a CUDA graph and replayed per step.

    One replay = network forward, fused V-trace/loss/grad kernel, network backward, [NCCL all-reduce],
    fused clip + optimizer update (any optim.FusedOptimizer), actor-weight publication: ~150 kernel launches
    become one cudaGraphLaunch, so a learner that reads its stats back every step (like the reference, monobeast.py:279-287) is no longer
    exposed to per-launch CPU latency.  Inputs are copied into static device buffers before each replay;
    the learning rate is read from a device scalar so LambdaLR keeps working; stats are computed from the
    graph's static outputs after the replay.

    The other values learn() reads (discounting, the two costs, reward clipping, the gradient clip, and the
    optimizer's alpha / eps / momentum / weight_decay / betas) are read from a device tb_hparams block that step()
    publishes before every replay, so they may change between steps without a new capture.  The values that choose a
    kernel or a buffer (`structure`) are fixed per graph; learn() captures another graph when one of them changes."""

    KEYS = ("frame", "reward", "done", "policy_logits", "action", "last_action", "episode_return", "task",
            "legal_actions")

    @staticmethod
    def structure_of(optimizer, batch, flags=None, model=None):
        """What the captured launch sequence depends on besides shapes: the optimizer's kernel and buffer choices
        (RMSprop centered / weight_decay != 0 / momentum != 0, Adam vs AdamW), the dtype of `done`, and whether
        `flags` turn the trust region, UPGO and kickstarting on (beta and the two costs are published per replay; on /
        off chooses the loss kernel, and UPGO and kickstarting add launches).  With kickstarting, the identity of
        `model`'s teacher net is part of it too: another teacher replays another graph."""
        trust = flags is not None and trust_region_kl(flags) is not None
        upgo = flags is not None and upgo_cost(flags) is not None
        ks = ()
        if flags is not None and kickstart_cost(flags) is not None:
            teacher = None if model is None else teacher_of(model)
            ks = ("kickstart", None if teacher is None else id(teacher.net))
        return (optimizer.structure() + (batch["done"].dtype,) + (("trust_region",) if trust else ())
                + (("upgo",) if upgo else ()) + ks)

    def __init__(self, flags, model, actor_model, optimizer, example_batch, initial_agent_state=()):
        _require_fused(optimizer)
        self.flags, self.model, self.actor, self.opt = flags, model, actor_model, optimizer
        self.structure = self.structure_of(optimizer, example_batch, flags, model)
        self.hparams = torch.zeros(HPARAMS.itemsize, dtype=torch.uint8, device=model.flat_params.device)
        publish_hparams(pack_hparams(flags, optimizer), self.hparams)
        # trust region: beta is a float32 device scalar published before every replay, like PopArt's beta
        self.trust_beta = None
        if trust_region_kl(flags) is not None:
            self.trust_beta = torch.zeros(1, dtype=torch.float32, device=model.flat_params.device)
            self._publish_trust_beta(flags)
        # UPGO: its cost is a float32 device scalar published before every replay, like the trust region's beta
        self.upgo_cost = None
        if upgo_cost(flags) is not None:
            self.upgo_cost = torch.zeros(1, dtype=torch.float32, device=model.flat_params.device)
            self._publish_upgo_cost(flags)
        # kickstarting: the cost is a device scalar published before every replay; the teacher is held so that its net
        # (whose identity keys this graph) and its zero states stay alive
        self.teacher = _teacher_for(model, actor_model, kickstart_cost(flags))
        self.kickstart_cost = None
        if self.teacher is not None:
            self.kickstart_cost = torch.zeros(1, dtype=torch.float32, device=model.flat_params.device)
            self._publish_kickstart_cost(flags)
        # PopArt: beta is a device scalar published before every replay, like the tb_hparams block
        self.popart = getattr(model, "popart", None)
        self.popart_beta = None
        if self.popart is not None:
            self.popart_beta = torch.zeros(1, dtype=torch.float64, device=model.flat_params.device)
            self._publish_beta(flags)
        self.static = {k: torch.empty_like(v) for k, v in example_batch.items() if k in self.KEYS}
        self.static_state = tuple(torch.empty_like(s) for s in initial_agent_state)
        for k, v in self.static.items():
            v.copy_(example_batch[k])
        for d, s in zip(self.static_state, initial_agent_state):
            d.copy_(s)
        optimizer.lr_from_device = True
        optimizer.sync_lr_to_device()
        # a replay buffer (model.replay): the mix runs inside the graph on the static fresh inputs, in the phase the buffer
        # is in now; learn() keeps one graph per phase
        _check_replay(model)
        self.replay = getattr(model, "replay", None)
        self.mixing = False
        replay_saved = None
        if self.replay is not None:
            self.fresh_columns = self.replay.prepare(self.static, self.static_state)
            self.mixing = self.replay.mixing(self.fresh_columns)
            replay_saved = self.replay.save(3)  # the two warm-up steps and the upload replay below each insert once
        # warm up on a side stream (allocations, one-time attribute calls), then capture
        self.obs_norm = getattr(model, "obs_norm", None)
        snapshot = (model.flat_params.clone(), optimizer.snapshot(),
                    None if self.popart is None else (self.popart.mu.clone(), self.popart.nu.clone()),
                    None if self.obs_norm is None else tuple(t.clone() for t in self.obs_norm.tensors()))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self._learn_step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = self._learn_step()
        # the graph writes into the model workspace it was captured with; the model replaces (and frees) that buffer when
        # it runs another shape, e.g. while the GraphedLearner of another batch shape is captured: keep it alive here
        self.workspace = getattr(model, "_ws", None)
        # the same holds for the stacked scratch an unstacked rollout is restacked into (AtariNet fp32, ResNet fp32 / bf16):
        # the graph writes it, its forward reads it, and the ResNet backward reads it again
        self.scratch = getattr(model, "_scratch_buf", None)
        # and for the teacher's workspace and restack scratch, which its forward in the graph writes
        self.teacher_workspace = self.teacher_scratch = None
        if self.teacher is not None:
            self.teacher_workspace = getattr(self.teacher.net, "_ws", None)
            self.teacher_scratch = getattr(self.teacher.net, "_scratch_buf", None)
        self.graph.replay()  # first replay uploads the graph to the device; keep that out of the training loop
        torch.cuda.synchronize()
        # undo the warm-up / capture-time updates so training starts from the caller's weights
        model.flat_params.copy_(snapshot[0])
        optimizer.restore(snapshot[1])  # state buffers and step count, the device step of Adam included
        if self.popart is not None:
            self.popart.mu.copy_(snapshot[2][0])
            self.popart.nu.copy_(snapshot[2][1])
        if self.obs_norm is not None:
            for dst, src in zip(self.obs_norm.tensors(), snapshot[3]):
                dst.copy_(src)
        if actor_model is not None and hasattr(actor_model, "copy_params_from"):
            actor_model.copy_params_from(model)
        if replay_saved is not None:
            self.replay.restore(replay_saved)  # ring slots, head, size, seed and step as the caller left them

    def _learn_step(self):
        """The captured launch sequence: [replay mix + advance], then learn_step without a host read."""
        batch, state = self.static, self.static_state
        draw = None
        if self.replay is not None:
            batch, state = self.replay.launch(batch, state, self.mixing)
            draw = self.replay.last_draw if self.replay.prioritized else None
        return learn_step(self.flags, self.model, self.actor, batch, state, self.opt, None, stats_sync=False,
                          hparams_dev=self.hparams, popart_beta_dev=self.popart_beta, draw=draw,
                          fresh_columns=self.fresh_columns if self.replay is not None else None,
                          trust_beta_dev=self.trust_beta, upgo_cost_dev=self.upgo_cost,
                          kickstart_cost_dev=self.kickstart_cost)

    def step(self, batch, initial_agent_state=(), scheduler=None, hparams=None):
        """One replay on `batch`.  `hparams`: the record of pack_hparams() to publish (default: packed from the
        flags this graph was captured with and the optimizer's current param group)."""
        for k, v in self.static.items():
            v.copy_(batch[k], non_blocking=True)
        for d, s in zip(self.static_state, initial_agent_state):
            d.copy_(s, non_blocking=True)
        self.opt.sync_lr_to_device()
        publish_hparams(pack_hparams(self.flags, self.opt) if hparams is None else hparams, self.hparams)
        if self.popart is not None:
            self._publish_beta(self.flags)
        if self.trust_beta is not None:
            self._publish_trust_beta(self.flags)
        if self.upgo_cost is not None:
            self._publish_upgo_cost(self.flags)
        if self.kickstart_cost is not None:
            self._publish_kickstart_cost(self.flags)
        if self.replay is not None:
            self.replay.prepare(self.static, self.static_state)  # publishes seed / step if the host changed them
        self.graph.replay()
        if self.replay is not None:
            self.replay.advance_host(self.fresh_columns)
        if scheduler is not None:
            scheduler.step()
        return self.out

    def _publish_beta(self, flags):
        """Enqueue the copy of flags.popart_beta into the device scalar through a fresh pinned buffer (publish_hparams)."""
        host = torch.full((1,), popart_beta(flags), dtype=torch.float64).pin_memory()
        self.popart_beta.copy_(host, non_blocking=True)

    def _publish_trust_beta(self, flags):
        """Enqueue the copy of flags.trust_region_kl (validated; float32) into the device scalar, as _publish_beta."""
        beta = trust_region_kl(flags)
        if beta is None:
            raise ValueError("this graph was captured with a trust region; trust_region_kl is now None")
        host = torch.full((1,), beta, dtype=torch.float32).pin_memory()
        self.trust_beta.copy_(host, non_blocking=True)

    def _publish_upgo_cost(self, flags):
        """Enqueue the copy of flags.upgo_cost (validated; float32) into the device scalar, as _publish_trust_beta."""
        cost = upgo_cost(flags)
        if cost is None:
            raise ValueError("this graph was captured with UPGO; upgo_cost is now None")
        host = torch.full((1,), cost, dtype=torch.float32).pin_memory()
        self.upgo_cost.copy_(host, non_blocking=True)

    def _publish_kickstart_cost(self, flags):
        """Enqueue the copy of flags.kickstart_cost (validated; float32) into the device scalar, as _publish_upgo_cost."""
        cost = kickstart_cost(flags)
        if cost is None:
            raise ValueError("this graph was captured with kickstarting; kickstart_cost is now None")
        host = torch.full((1,), cost, dtype=torch.float32).pin_memory()
        self.kickstart_cost.copy_(host, non_blocking=True)

    def _losses_out(self):
        """The step's loss values, then the trust-region sums, the UPGO loss and the kickstarting loss and KL sum when
        on: float32 [4] to [9]."""
        return _loss_values(self.out["losses"], self.out["trust"], self.out["upgo"], self.out["kickstart"])

    def _kickstart_rows(self):
        return _kickstart_rows(self.out["kickstart"], self.out["vtrace"])

    def snapshot(self):
        """Device copies of what stats() reads (the step's losses and its done / episode_return rows, a PopArt model's
        statistics, the trust-region sums and row count, the UPGO loss, the kickstarting values), enqueued on the current stream: lets the caller
        release the learner lock BEFORE the blocking read-back, so the next learner thread's replay queues up behind
        this one instead of waiting for a host round trip."""
        trust = self.out["trust"]
        snap = (self._losses_out(), self.static["done"][1:].clone(), self.static["episode_return"][1:].clone(),
                None if trust is None else trust.kl.numel(), self.out["upgo"] is not None, self._kickstart_rows())
        if self.popart is not None:
            snap += (self.popart.mu.clone(), self.popart.nu.clone())
        return snap

    _tls = threading.local()

    @staticmethod
    def stats_from(snap, event):
        """Read the snapshot back on a per-thread READ-BACK stream that waits only for `event` (recorded right after the
        snapshot): a read-back on the compute stream would queue behind the NEXT step, which another learner thread has
        already enqueued there."""
        losses, done, ep_ret, trust_rows, has_upgo, kickstart_rows = snap[:6]
        tls = GraphedLearner._tls
        dev = losses.device
        if getattr(tls, "stream", None) is None or tls.device != dev:
            tls.stream, tls.device, tls.pinned = torch.cuda.Stream(device=dev), dev, {}
        key = (tuple(done.shape), done.dtype, losses.numel())
        bufs = tls.pinned.get(key)
        if bufs is None:
            bufs = tls.pinned[key] = (torch.empty(losses.numel(), dtype=torch.float32).pin_memory(),
                                      torch.empty(done.shape, dtype=done.dtype).pin_memory(),
                                      torch.empty(ep_ret.shape, dtype=ep_ret.dtype).pin_memory())
        tls.stream.wait_event(event)
        with torch.cuda.stream(tls.stream):
            for dst, src in zip(bufs, (losses, done, ep_ret)):
                dst.copy_(src, non_blocking=True)
            popart = [s.to("cpu", non_blocking=True) for s in snap[6:]]
        tls.stream.synchronize()
        host, hdone, hret = bufs
        ep = hret[hdone.bool()].clone()
        stats = {
            "episode_returns": tuple(ep.numpy()), "mean_episode_return": torch.mean(ep).item(),
            "total_loss": host[3].item(), "pg_loss": host[0].item(), "baseline_loss": host[1].item(),
            "entropy_loss": host[2].item(),
        }
        stats.update(_extra_stats(host, trust_rows, has_upgo, kickstart_rows))
        if popart:
            stats.update(_popart_stats(*popart))
        return stats

    def stats(self):
        """Same keys as monobeast.learn()'s return value; one blocking read-back."""
        done = self.static["done"][1:]
        ep = self.static["episode_return"][1:][done.bool()].cpu()
        host = self._losses_out().cpu()
        stats = {
            "episode_returns": tuple(ep.numpy()), "mean_episode_return": torch.mean(ep).item(),
            "total_loss": host[3].item(), "pg_loss": host[0].item(), "baseline_loss": host[1].item(),
            "entropy_loss": host[2].item(),
        }
        trust = self.out["trust"]
        stats.update(_extra_stats(host, None if trust is None else trust.kl.numel(), self.out["upgo"] is not None,
                                  self._kickstart_rows()))
        if self.popart is not None:
            stats.update(_popart_stats(self.popart.mu.cpu(), self.popart.nu.cpu()))
        return stats
