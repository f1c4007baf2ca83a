"""Time the graphed learn step (monobeast.learn with flags.cuda_graph) at T=80, B=32, AtariNet + LSTM, default backend,
without PopArt, with PopArt at one task and at 57 tasks (column b plays task b mod 57), in alternating rounds; every
leg trains on unclipped rewards.  Prints the card and its power limit.

    python tools/bench_popart.py [--rounds 3] [--steps 50]
"""
import argparse
import os
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import monobeast, optim  # noqa: E402

T, B, A = 80, 32, 6


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def learner(num_tasks):
    model = monobeast.AtariNet((4, 84, 84), A, True, num_tasks=num_tasks)
    actor = monobeast.AtariNet((4, 84, 84), A, True, num_tasks=num_tasks)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="none", discounting=0.99,
                                  baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=True,
                                  popart_beta=3e-4)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=2).items()}
    if num_tasks:
        batch["task"] = (torch.arange(B, device="cuda") % num_tasks).expand(T + 1, B).contiguous()
    state = model.initial_state(B)
    return lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_popart needs a GPU")
    legs = {"no PopArt": learner(None), "PopArt, K=1": learner(1), "PopArt, K=57": learner(57)}
    for step in legs.values():
        for _ in range(5):
            step()
    torch.cuda.synchronize()
    print("card: %s" % card())
    for r in range(args.rounds):
        for name, step in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step()  # reads its stats back: one host sync per step, as in training
            torch.cuda.synchronize()
            print("round %d  %-12s %.3f ms/step" % (r, name, (time.perf_counter() - t0) * 1e3 / args.steps))


if __name__ == "__main__":
    main()
