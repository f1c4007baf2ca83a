"""Fused pieces of the learner step shared by monobeast.learn and polybeast_learner.learn."""
import collections
import os
import threading

import torch

from torchbeast_b200 import _lib

ImpalaLoss = collections.namedtuple(
    "ImpalaLoss",
    "vs pg_advantages log_rhos behavior_action_log_probs target_action_log_probs losses grad_logits grad_values",
)


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
):
    """The whole loss block of learn() in ONE kernel launch (tb_impala_loss_fwd_bwd_f32).

    Inputs are the shifted [T,B,...] slices (batch[1:], learner_outputs[:-1]); `done` is a
    bool/uint8 tensor.  Replaces monobeast.py:245-277 / polybeast_learner.py:332-361 and the
    autograd graph behind them: returns vs / pg_advantages / log-rhos, losses =
    [pg, baseline_cost*baseline, entropy_cost*entropy, total] and d total / d(target logits,
    values) laid out as [T+1,B,...] with a zero bootstrap row, ready for the network backward.
    """
    tensors = (behavior_policy_logits, target_policy_logits, actions, rewards, done, values, bootstrap_value)
    _lib.require_cuda(*tensors)
    if reward_clipping not in ("abs_one", "none"):
        raise ValueError("reward_clipping must be 'abs_one' or 'none'")
    T, B, A = target_policy_logits.shape
    dev = values.device
    f32 = torch.float32
    bl = behavior_policy_logits.to(f32).contiguous()
    tl = target_policy_logits.detach().to(f32).contiguous()
    ac = actions.to(torch.int64).contiguous()
    rw = rewards.to(f32).contiguous()
    if done.dtype == torch.bool:
        dn = done.contiguous().view(torch.uint8)
        disc = None
    elif done.dtype == torch.uint8:
        # `~done` on uint8 is a bitwise NOT in the reference (SURVEY Appendix A): discount = (255-done)*gamma
        dn, disc = None, ((~done).to(f32) * discounting).contiguous()
    else:
        raise _lib.TorchBeastB200Error("done must be bool or uint8")
    va = values.detach().to(f32).contiguous()
    bs = bootstrap_value.detach().to(f32).contiguous()
    outs = [torch.empty((T, B), dtype=f32, device=dev) for _ in range(5)]
    losses = torch.empty(4, dtype=f32, device=dev)
    gl = torch.empty((T + 1, B, A), dtype=f32, device=dev) if with_grads else None
    gv = torch.empty((T + 1, B), dtype=f32, device=dev) if with_grads else None
    _lib.check(
        _lib.lib().tb_impala_loss_fwd_bwd_f32(
            _lib.ptr(bl), _lib.ptr(tl), _lib.ptr(ac), _lib.ptr(rw), _lib.ptr(dn), _lib.ptr(disc),
            _lib.ptr(va), _lib.ptr(bs), T, B, A, float(discounting), float(baseline_cost), float(entropy_cost),
            int(reward_clipping == "abs_one"), _lib.clip_arg(clip_rho_threshold), _lib.clip_arg(clip_pg_rho_threshold),
            *[_lib.ptr(o) for o in outs], _lib.ptr(losses), _lib.ptr(gl), _lib.ptr(gv), 1,
            _lib.ptr(_lib.workspace()), _lib.stream_ptr()),
        "tb_impala_loss_fwd_bwd_f32")
    vs, pg, lr, blp, tlp = outs
    return ImpalaLoss(vs, pg, lr, blp, tlp, losses, gl, gv)


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


def optimizer_step(model, optimizer, max_grad_norm):
    from torchbeast_b200 import optim as _optim

    if isinstance(optimizer, _optim.RMSprop):
        optimizer.step(max_grad_norm=max_grad_norm)  # fused clip + RMSprop, 2 launches
    else:
        # foreign optimizer object: gradients are already in .grad (views of the flat buffer)
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)
        optimizer.step()


def learn_step(flags, model, actor_model, batch, initial_agent_state, optimizer, scheduler,
               behavior_logits=None, actions=None, stats_sync=True):
    """One optimisation step on a [T+1, B, ...] rollout batch (dict of CUDA tensors).

    Launch sequence (no autograd graph, no host sync until the stats read-back):
      network forward -> fused V-trace + 3 losses + their gradients (1 launch) -> network
      backward into the flat gradient -> [NCCL all-reduce] -> fused clip + RMSprop -> actor copy.
    """
    out = model.learner_forward(batch, initial_agent_state)
    blogits = batch["policy_logits"] if behavior_logits is None else behavior_logits
    acts = batch["action"] if actions is None else actions
    loss = impala_loss_fwd_bwd(
        blogits[1:], out.policy_logits[:-1], acts[1:], batch["reward"][1:], batch["done"][1:],
        out.baseline[:-1], out.baseline[-1],
        discounting=flags.discounting, baseline_cost=flags.baseline_cost, entropy_cost=flags.entropy_cost,
        reward_clipping=flags.reward_clipping)
    _backward_with_overlapped_all_reduce(model, loss.grad_logits, loss.grad_values)
    optimizer_step(model, optimizer, flags.grad_norm_clipping)
    if scheduler is not None:
        scheduler.step()
    if actor_model is not None and actor_model is not model:
        if hasattr(actor_model, "copy_params_from") and hasattr(model, "flat_params"):
            actor_model.copy_params_from(model)
        else:
            actor_model.load_state_dict(model.state_dict())
    if not stats_sync:
        return dict(losses=loss.losses, vtrace=loss)
    done = batch["done"][1:]
    episode_returns = batch["episode_return"][1:][done.bool()]
    host = loss.losses.cpu()  # the step's one blocking read-back
    ep = episode_returns.cpu()
    return {
        "episode_returns": tuple(ep.numpy()),
        "mean_episode_return": torch.mean(ep).item(),
        "total_loss": host[3].item(),
        "pg_loss": host[0].item(),
        "baseline_loss": host[1].item(),
        "entropy_loss": host[2].item(),
    }


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
    Returns the reference's stats dict."""
    import contextlib
    from torchbeast_b200 import staging
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
        if "last_action" not in batch and getattr(model, "needs_last_action", False):
            # the polybeast nest has no separate last_action leaf: row t of `action` IS the action taken before frame t
            batch = dict(batch, last_action=batch["action"])
        try:
            if _graph_enabled(flags):
                graphs = model.__dict__.setdefault("_tb_graphs", {})
                gkey = (tuple((k, tuple(v.shape)) for k, v in batch.items() if k in GraphedLearner.KEYS), id(optimizer),
                        id(actor_model))
                gl = graphs.get(gkey)
                if gl is None:
                    gl = graphs[gkey] = GraphedLearner(flags, model, actor_model, optimizer, batch, initial_agent_state)
                gl.step(batch, initial_agent_state, scheduler)
                if stager is not None:
                    stager.release(slot)  # the inputs now live in the graph's static buffers
                    slot = None
                if os.environ.get("TB_STATS_IN_LOCK", "0") == "1":   # the reference's behaviour: read back under the lock
                    return gl.stats()
                snap = gl.snapshot()      # tiny device copies, still under the lock (the next replay overwrites the originals)
                snap_event = torch.cuda.Event()
                snap_event.record()
            else:
                return learn_step(flags, model, actor_model, batch, initial_agent_state, optimizer, scheduler)
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


class GraphedLearner:
    """The whole device side of learn() captured ONCE into a CUDA graph and replayed per step.

    One replay = network forward, fused V-trace/loss/grad kernel, network backward, [NCCL all-reduce],
    fused clip + RMSprop, actor-weight publication: ~150 kernel launches become one cudaGraphLaunch, so
    a learner that reads its stats back every step (like the reference, monobeast.py:279-287) is no longer
    exposed to per-launch CPU latency.  Inputs are copied into static device buffers before each replay;
    the learning rate is read from a device scalar so LambdaLR keeps working; stats are computed from the
    graph's static outputs after the replay."""

    KEYS = ("frame", "reward", "done", "policy_logits", "action", "last_action", "episode_return")

    def __init__(self, flags, model, actor_model, optimizer, example_batch, initial_agent_state=()):
        from torchbeast_b200 import optim as _optim
        if not isinstance(optimizer, _optim.RMSprop):
            raise _lib.TorchBeastB200Error("GraphedLearner needs torchbeast_b200.optim.RMSprop")
        self.flags, self.model, self.actor, self.opt = flags, model, actor_model, optimizer
        self.static = {k: torch.empty_like(v) for k, v in example_batch.items() if k in self.KEYS}
        self.static_state = tuple(torch.empty_like(s) for s in initial_agent_state)
        for k, v in self.static.items():
            v.copy_(example_batch[k])
        for d, s in zip(self.static_state, initial_agent_state):
            d.copy_(s)
        optimizer.lr_from_device = True
        optimizer.sync_lr_to_device()
        # warm up on a side stream (allocations, one-time attribute calls), then capture
        snapshot = (model.flat_params.clone(), optimizer.square_avg.clone(),
                    None if optimizer.momentum_buffer is None else optimizer.momentum_buffer.clone(), optimizer._steps)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                learn_step(flags, model, actor_model, self.static, self.static_state, optimizer, None, stats_sync=False)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = learn_step(flags, model, actor_model, self.static, self.static_state, optimizer, None,
                                  stats_sync=False)
        # the graph writes into the model workspace it was captured with; the model replaces (and frees) that buffer when
        # it runs another shape, e.g. while the GraphedLearner of another batch shape is captured: keep it alive here
        self.workspace = getattr(model, "_ws", None)
        self.graph.replay()  # first replay uploads the graph to the device; keep that out of the training loop
        torch.cuda.synchronize()
        # undo the warm-up / capture-time updates so training starts from the caller's weights
        model.flat_params.copy_(snapshot[0])
        optimizer.square_avg.copy_(snapshot[1])
        if snapshot[2] is not None:
            optimizer.momentum_buffer.copy_(snapshot[2])
        optimizer._steps = snapshot[3]
        if actor_model is not None and hasattr(actor_model, "copy_params_from"):
            actor_model.copy_params_from(model)

    def step(self, batch, initial_agent_state=(), scheduler=None):
        for k, v in self.static.items():
            v.copy_(batch[k], non_blocking=True)
        for d, s in zip(self.static_state, initial_agent_state):
            d.copy_(s, non_blocking=True)
        self.opt.sync_lr_to_device()
        self.graph.replay()
        if scheduler is not None:
            scheduler.step()
        return self.out

    def snapshot(self):
        """Device copies of what stats() reads (the step's losses and its done / episode_return rows), enqueued on the
        current stream: lets the caller release the learner lock BEFORE the blocking read-back, so the next learner
        thread's replay queues up behind this one instead of waiting for a host round trip."""
        return (self.out["losses"].clone(), self.static["done"][1:].clone(), self.static["episode_return"][1:].clone())

    _tls = threading.local()

    @staticmethod
    def stats_from(snap, event):
        """Read the snapshot back on a per-thread READ-BACK stream that waits only for `event` (recorded right after the
        snapshot): a read-back on the compute stream would queue behind the NEXT step, which another learner thread has
        already enqueued there."""
        losses, done, ep_ret = snap
        tls = GraphedLearner._tls
        dev = losses.device
        if getattr(tls, "stream", None) is None or tls.device != dev:
            tls.stream, tls.device, tls.pinned = torch.cuda.Stream(device=dev), dev, {}
        key = (tuple(done.shape), done.dtype)
        bufs = tls.pinned.get(key)
        if bufs is None:
            bufs = tls.pinned[key] = (torch.empty(4, dtype=torch.float32).pin_memory(), torch.empty(done.shape, dtype=done.dtype).pin_memory(),
                                      torch.empty(ep_ret.shape, dtype=ep_ret.dtype).pin_memory())
        tls.stream.wait_event(event)
        with torch.cuda.stream(tls.stream):
            for dst, src in zip(bufs, (losses, done, ep_ret)):
                dst.copy_(src, non_blocking=True)
        tls.stream.synchronize()
        host, hdone, hret = bufs
        ep = hret[hdone.bool()].clone()
        return {
            "episode_returns": tuple(ep.numpy()), "mean_episode_return": torch.mean(ep).item(),
            "total_loss": host[3].item(), "pg_loss": host[0].item(), "baseline_loss": host[1].item(),
            "entropy_loss": host[2].item(),
        }

    def stats(self):
        """Same keys as monobeast.learn()'s return value; one blocking read-back."""
        done = self.static["done"][1:]
        ep = self.static["episode_return"][1:][done.bool()].cpu()
        host = self.out["losses"].cpu()
        return {
            "episode_returns": tuple(ep.numpy()), "mean_episode_return": torch.mean(ep).item(),
            "total_loss": host[3].item(), "pg_loss": host[0].item(), "baseline_loss": host[1].item(),
            "entropy_loss": host[2].item(),
        }
