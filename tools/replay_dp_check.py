"""Two data-parallel ranks, each with its own replay buffer (stream id = rank), keep bit-identical replicas.

    python -m torch.distributed.run --nproc-per-node 2 tools/replay_dp_check.py

Each rank learns 3 steps on its own batches (1 warm-up step, 2 mixing steps); rank 0 prints one JSON line:
replicas_bit_identical (the flat parameters agree bit for bit) and slots_differ (the ranks drew different slots)."""
import json
import os
import sys
import types

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import learner, monobeast, optim  # noqa: E402
from torchbeast_b200.replay import ReplayBuffer  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl")
    T, Bf, A = 4, 4, 6
    model, actor = (monobeast.AtariNet((4, 84, 84), A, True) for _ in range(2))
    model.reset_parameters_like_torch(seed=3)
    actor.copy_params_from(model)
    model.replay = ReplayBuffer(12, 4, seed=5, min_size=4)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006,
                                  grad_norm_clipping=40.0)
    for k in range(3):
        batch = {key: v.cuda() for key, v in LT.synthetic_batch(T, Bf, A, seed=100 * rank + k).items()}
        learner.learn(flags, model, actor, batch, model.initial_state(Bf), opt, None)
    torch.cuda.synchronize()
    params = [torch.empty_like(model.flat_params) for _ in range(world)]
    dist.all_gather(params, model.flat_params)
    slots = [torch.empty_like(model.replay.last_slots) for _ in range(world)]
    dist.all_gather(slots, model.replay.last_slots)
    if rank == 0:
        print(json.dumps({"replicas_bit_identical": all(torch.equal(params[0], p) for p in params[1:]),
                          "slots_differ": any(not torch.equal(slots[0], s) for s in slots[1:])}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
