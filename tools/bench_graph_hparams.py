"""Cost of following hyper-parameter changes in the graphed learner, measured in alternating rounds.

    python tools/bench_graph_hparams.py [--rounds 3] [--steps 100] [--T 80] [--B 32]

Per round it reports, for the graphed monobeast.learn step (AtariNet + LSTM, default backend, reference RMSprop,
flags.cuda_graph, device-resident batch, stats read back every step):
  * learn_ms, values constant: the same flags and param group every step;
  * learn_ms, values changing: entropy_cost, baseline_cost, discounting, grad_norm_clipping and RMSprop's alpha / eps
    change before every step (the lr follows a LambdaLR in both);
  * host_us: host time of one GraphedLearner.step call (input copies, lr and hyper-parameter publication, replay
    launch) and of pack_hparams + publish_hparams alone, averaged over `--steps` calls that each start on an idle GPU.
CUDA events around `--steps` steps after the capture and a warm-up.  The card's name and power limit are printed first:
the numbers belong to them.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import learner, monobeast, optim  # noqa: E402

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)
A = 6


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (torch.cuda.get_device_name(0), q)


def vary(k, flags, opt):
    """Small per-step changes around the reference values (the gradient clip stays in use)."""
    flags.entropy_cost = 0.0006 * (1.0 + 0.01 * (k % 7))
    flags.baseline_cost = 0.5 - 0.001 * (k % 5)
    flags.discounting = 0.99 - 1e-4 * (k % 3)
    flags.grad_norm_clipping = 40.0 - 0.1 * (k % 4)
    g = opt.param_groups[0]
    g["alpha"] = 0.99 - 1e-4 * (k % 6)
    g["eps"] = 0.01 * (1.0 + 0.01 * (k % 5))


class Setup:
    def __init__(self, T, B):
        self.model = monobeast.AtariNet((4, 84, 84), A, True)
        self.actor = monobeast.AtariNet((4, 84, 84), A, True)
        self.model.reset_parameters_like_torch(seed=1)
        self.actor.copy_params_from(self.model)
        self.opt = optim.RMSprop(self.model, lr=0.00048, momentum=0, eps=0.01, alpha=0.99)
        self.sched = torch.optim.lr_scheduler.LambdaLR(self.opt, lambda e: 1 - min(e * T * B, 30_000_000) / 30_000_000)
        self.flags = types.SimpleNamespace(unroll_length=T, batch_size=B, cuda_graph=True, **FLAGS)
        self.batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=2).items()}
        self.state = tuple(torch.zeros(2, B, 512 + A + 1, device="cuda") for _ in range(2))
        self.k = 0

    def learn(self, changing):
        if changing:
            vary(self.k, self.flags, self.opt)
        self.k += 1
        return monobeast.learn(self.flags, self.actor, self.model, self.batch, self.state, self.opt, self.sched)

    def graph(self):
        (gl,) = [g for key, g in self.model._tb_graphs.items() if len(key) == 3]
        return gl


def learn_ms(setup, changing, steps, warmup=5):
    for _ in range(warmup):
        setup.learn(changing)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        setup.learn(changing)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def host_us(setup, steps):
    """Host time of one call, each call starting on an idle GPU (so no call waits for a full launch queue)."""
    gl = setup.graph()
    step_s = publish_s = 0.0
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gl.step(setup.batch, setup.state, setup.sched)
        step_s += time.perf_counter() - t0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        learner.publish_hparams(learner.pack_hparams(setup.flags, setup.opt), gl.hparams)
        publish_s += time.perf_counter() - t0
    torch.cuda.synchronize()
    return 1e6 * step_s / steps, 1e6 * publish_s / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=80)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_hparams measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    print("card: %s" % card(), flush=True)
    setup = Setup(args.T, args.B)
    setup.learn(False)  # capture
    for r in range(args.rounds):
        for changing in ((False, True) if r % 2 == 0 else (True, False)):
            ms = learn_ms(setup, changing, args.steps)
            print(json.dumps(dict(round=r, bench="graphed learn", T=args.T, B=args.B, values="changing" if changing
                                  else "constant", learn_ms=round(ms, 4))), flush=True)
        step_us, publish_us = host_us(setup, args.steps)
        print(json.dumps(dict(round=r, bench="host", step_us=round(step_us, 1), pack_publish_us=round(publish_us, 1))),
              flush=True)
    assert len(setup.model._tb_graphs) == 1  # every change reused the one graph


if __name__ == "__main__":
    main()
