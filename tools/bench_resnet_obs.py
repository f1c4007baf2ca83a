"""Time the graphed learn step of the IMPALA ResNet (polybeast_learner.Net + LSTM, default bf16x3 backend,
learner.learn with flags.cuda_graph) at T=80 and B = 8 and 32 for the Atari stack (4, 84, 84), Procgen (3, 64, 64) and
DMLab (3, 72, 96) observations, in alternating rounds.  Prints the card and its power limit, then ms/step and learner
frames/s (T x B environment frames per step, as stats["step"] counts them) per shape.

    python tools/bench_resnet_obs.py [--rounds 3] [--steps 30]
"""
import argparse
import os
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import learner, optim, polybeast_learner  # noqa: E402

T, A = 80, 6
SHAPES = [(4, 84, 84), (3, 64, 64), (3, 72, 96)]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def leg(obs, B):
    model = polybeast_learner.Net(A, True, observation_shape=obs)
    actor = polybeast_learner.Net(A, True, observation_shape=obs)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006,
                                  grad_norm_clipping=40.0, cuda_graph=True)
    batch = LT.synthetic_batch(T, B, A, seed=2, with_last_action=False)
    batch["frame"] = torch.from_numpy(np.random.RandomState(3).randint(0, 256, size=(T + 1, B) + obs).astype(np.uint8))
    batch = {k: v.cuda() for k, v in batch.items()}
    state = model.initial_state(B)
    return lambda: learner.learn(flags, model, actor, batch, state, opt, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--batch-sizes", default="8,32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resnet_obs needs a GPU")
    sizes = [int(b) for b in args.batch_sizes.split(",")]
    legs = {(obs, B): leg(obs, B) for B in sizes for obs in SHAPES}
    for step in legs.values():
        for _ in range(5):   # the graph capture and its warm-up
            step()
    torch.cuda.synchronize()
    print("card: %s" % card())
    for r in range(args.rounds):
        for (obs, B), step in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step()  # reads its stats back: one host sync per step, as in training
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / args.steps
            print("round %d  obs %-12s B=%-3d %8.3f ms/step %10.0f frames/s"
                  % (r, "%dx%dx%d" % obs, B, ms, T * B / ms * 1e3), flush=True)


if __name__ == "__main__":
    main()
