"""CUDA drop-in for the learner-side symbols of torchbeast/polybeast_learner.py.

Exports (same names/signatures as /root/reference/torchbeast/polybeast_learner.py):
  compute_baseline_loss / compute_entropy_loss / compute_policy_gradient_loss   :113-131
  learn(flags, learner_queue, model, actor_model, optimizer, scheduler, stats, plogger, lock) :295-389
ActorPool / DynamicBatcher / gRPC env server / train() orchestration are out of scope
(SURVEY.md 2); learn() consumes the same ((env_outputs, actor_outputs), initial_agent_state)
nest that learner_queue yields (SURVEY.md 8(b) B2).
"""
from torchbeast_b200.losses import (  # noqa: F401
    compute_baseline_loss,
    compute_entropy_loss,
    compute_policy_gradient_loss,
)

import collections  # noqa: E402
import os  # noqa: E402
import threading  # noqa: E402

import torch  # noqa: E402

from torchbeast_b200 import acting as _acting  # noqa: E402
from torchbeast_b200 import learner as _learner  # noqa: E402
from torchbeast_b200.nets import ResNet as Net  # noqa: E402,F401

EnvOutput = collections.namedtuple("EnvOutput", "frame rewards done episode_step episode_return")
AgentOutput = collections.namedtuple("AgentOutput", "action policy_logits baseline")
Batch = collections.namedtuple("Batch", "env agent")


def _map_nest(fn, n):
    """nest.map for the tuple / list / dict nests the reference passes around (nest_pybind.h:61-67: vectors are tuples)."""
    if isinstance(n, torch.Tensor):
        return fn(n)
    if isinstance(n, dict):
        return {k: _map_nest(fn, v) for k, v in n.items()}
    return tuple(_map_nest(fn, v) for v in n)


def inference(flags, inference_batcher, model, lock=threading.Lock()):  # noqa: B008
    """The inference thread body - reference polybeast_learner.py:269-285 (SURVEY 8(f) N2).

    `inference_batcher` yields DynamicBatcher batches (actorpool.cc:224-340): `batch.get_inputs()` returns
    `(batched_env_outputs, agent_state)` with [T=1, B, ...] leaves, B = 1 .. 512 actors; the forward of the SAME CUDA
    kernels the learner uses runs under `lock` on flags.actor_device, and `batch.set_outputs(((action, policy_logits,
    baseline), core_state))` receives CPU tensors, like the reference.  Works for polybeast's Net (ResNet) and for AtariNet
    (whose `last_action` input is batched_env_outputs[5] if the nest carries one, else zeros).

    A sampler attached as `model.action_sampler` (torchbeast_b200.sampling) replaces torch.multinomial in training mode;
    its step advances by one per call, safely across inference threads because the forward runs under `lock`.  The
    polybeast nest carries no actor id, so each row's stream id is its index in the batch: a run is reproducible for a
    given sequence of batches, not per actor.

    With flags.inference_graph (or TB_INFERENCE_GRAPH=1) the forward is a CUDA-graph replay (torchbeast_b200.acting.
    GraphedActor, one per model, shared by the inference threads); training mode then needs a sampler attached.  The
    replay's outputs live in the graph's static buffers, which the next thread's replay overwrites, so their copy to
    the host is enqueued before the lock is released."""
    device = torch.device(getattr(flags, "actor_device", None) or model.flat_params.device)
    graphed = inference_graph_enabled(flags)
    with torch.no_grad():
        for batch in inference_batcher:
            batched_env_outputs, agent_state = batch.get_inputs()
            frame, reward, done, *rest = batched_env_outputs
            inputs = dict(frame=frame.to(device, non_blocking=True), reward=reward.to(device, non_blocking=True),
                          done=done.to(device, non_blocking=True))
            if getattr(model, "needs_last_action", False):
                la = rest[2] if len(rest) > 2 else torch.zeros(reward.shape, dtype=torch.int64)
                inputs["last_action"] = la.to(device, non_blocking=True)
            agent_state = _map_nest(lambda t: t.to(device, non_blocking=True), agent_state)
            if graphed:
                with lock:
                    actor = model.__dict__.get("_tb_graphed_actor")
                    if actor is None:
                        actor = model._tb_graphed_actor = _acting.GraphedActor(model)
                    host = _map_nest(_to_pinned_async, _net_outputs(actor(inputs, agent_state)))
                    ready = torch.cuda.Event()
                    ready.record()
                ready.synchronize()
                batch.set_outputs(host)
                continue
            with lock:
                outputs = model(inputs, agent_state)
            outputs = _net_outputs(outputs)
            batch.set_outputs(_map_nest(lambda t: t.cpu(), outputs))


def inference_graph_enabled(flags):
    """The graphed inference forward is opt-in: flags.inference_graph (or TB_INFERENCE_GRAPH=1)."""
    v = getattr(flags, "inference_graph", None)
    if v is None:
        v = os.environ.get("TB_INFERENCE_GRAPH", "0") not in ("0", "", "false")
    return bool(v)


def _net_outputs(outputs):
    if isinstance(outputs[0], dict):  # AtariNet returns a dict (monobeast.py:626-632): same tuple order as Net
        o = outputs[0]
        outputs = ((o["action"], o["policy_logits"], o["baseline"]), outputs[1])
    return outputs


def _to_pinned_async(t):
    """A fresh pinned host tensor receiving `t` by a copy enqueued on the current stream (the caching host allocator
    does not hand the block out again while the copy is pending)."""
    return torch.empty(t.shape, dtype=t.dtype, pin_memory=True).copy_(t, non_blocking=True)


def _to_device(t, device):
    return t.to(device, non_blocking=True) if isinstance(t, torch.Tensor) else t


def learn(
    flags,
    learner_queue,
    model,
    actor_model,
    optimizer,
    scheduler,
    stats,
    plogger,
    lock=threading.Lock(),  # noqa: B008
):
    """The learner thread body - reference polybeast_learner.py:295-389.

    Consumes the same nest the reference's BatchingQueue yields (SURVEY.md 8(b) B2):
    ((env_outputs, actor_outputs), initial_agent_state) with [T+1, B, ...] CPU (or CUDA) leaves,
    env_outputs = (frame u8, reward, done, episode_step, episode_return), actor_outputs =
    (action, policy_logits, baseline); fills `stats` with the reference's keys and calls plogger.log."""
    for tensors in learner_queue:
        batch, initial_agent_state = tensors
        env_outputs, actor_outputs = batch
        env = EnvOutput._make(list(env_outputs)[:5])
        agent = AgentOutput._make(list(actor_outputs)[:3])
        rollout = dict(frame=env.frame, reward=env.rewards, done=env.done, episode_return=env.episode_return,
                       episode_step=env.episode_step, policy_logits=agent.policy_logits, action=agent.action)
        # host nest (what the reference's BatchingQueue yields) -> pinned slot -> async H2D, OUTSIDE the lock: with
        # num_learner_threads = 2 (polybeast_learner.py:62,505-521) this thread's copy overlaps the other thread's step.
        # _learner.learn takes the lock for the step itself (only one thread learning at a time, pl:313).
        mean_step = torch.mean(env.episode_step[1:].float()).item()
        out = _learner.learn(flags, model, actor_model, rollout, tuple(initial_agent_state), optimizer, scheduler, lock)
        with lock:
            stats["step"] = stats.get("step", 0) + flags.unroll_length * flags.batch_size
            stats["episode_returns"] = out["episode_returns"]
            stats["mean_episode_return"] = out["mean_episode_return"]
            stats["mean_episode_step"] = mean_step
            for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
                stats[k] = out[k]
            stats["learner_queue_size"] = learner_queue.size()
            plogger.log(stats)
            if not len(out["episode_returns"]):
                stats["mean_episode_return"] = None  # hide the mean-of-empty NaN, like the reference
