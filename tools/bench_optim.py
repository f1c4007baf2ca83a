"""Cost of the fused optimizer steps on one GPU, each comparison measured in alternating rounds.

    python tools/bench_optim.py [--rounds 3] [--steps 50] [--T 80] [--B 32]

Per round it reports:
  * optim_ms: one clip + Adam step over the AtariNet flat buffers, P = 6.0 M (with LSTM) and 1.69 M (without):
    torchbeast_b200.optim.Adam.step(max_grad_norm=40) (tb_grad_sumsq_f32 + tb_clip_adam_step_f32) against
    torch.nn.utils.clip_grad_norm_(foreach=True) + torch.optim.Adam(fused=True) over the same 20 (12 without LSTM)
    parameter views.  CUDA events around `--steps` steps after a warm-up.
  * learn_ms: the graphed monobeast.learn step (AtariNet + LSTM, default backend, flags.cuda_graph, device-resident
    batch, stats read back every step) with optim.RMSprop against the same step with optim.Adam.  CUDA events around
    `--steps` steps after the capture and a warm-up.
The card's name and power limit are printed first: the numbers belong to them.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import monobeast, optim  # noqa: E402

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)
A = 6


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (torch.cuda.get_device_name(0), q)


def timed(fn, steps, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def optim_step(impl, use_lstm, steps):
    model = monobeast.AtariNet((4, 84, 84), A, use_lstm)
    model.reset_parameters_like_torch(seed=1)
    grad = model.attach_grads()
    grad.copy_(torch.randn_like(grad) * (80.0 / grad.numel() ** 0.5))  # norm 80: the clip at 40 is active
    if impl == "fused":
        opt = optim.Adam(model, lr=1e-4)
        step = lambda: opt.step(max_grad_norm=40.0)  # noqa: E731
    else:
        params = list(model.parameters())
        opt = torch.optim.Adam(params, lr=1e-4, fused=True)

        def step():
            torch.nn.utils.clip_grad_norm_(params, 40.0, foreach=True)
            opt.step()
    return model.flat_params.numel(), len(list(model.parameters())), timed(step, steps)


def learn_step(name, T, B, steps):
    model = monobeast.AtariNet((4, 84, 84), A, True)
    actor = monobeast.AtariNet((4, 84, 84), A, True)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99) if name == "rmsprop" else optim.Adam(model, lr=1e-4)
    flags = types.SimpleNamespace(unroll_length=T, batch_size=B, cuda_graph=True, **FLAGS)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=2).items()}
    state = tuple(torch.zeros(2, B, 512 + A + 1, device="cuda") for _ in range(2))
    return timed(lambda: monobeast.learn(flags, actor, model, batch, state, opt, None), steps, warmup=3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=80)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    print("card: %s" % card(), flush=True)
    for r in range(args.rounds):
        for use_lstm in (True, False):
            for impl in ("fused", "torch"):
                P, views, ms = optim_step(impl, use_lstm, args.steps)
                print(json.dumps(dict(round=r, bench="clip+adam", impl=impl, params=P, views=views,
                                      optim_ms=round(ms, 4))), flush=True)
        for name in ("rmsprop", "adam"):
            ms = learn_step(name, args.T, args.B, args.steps)
            print(json.dumps(dict(round=r, bench="graphed learn", T=args.T, B=args.B, optimizer=name,
                                  learn_ms=round(ms, 3))), flush=True)


if __name__ == "__main__":
    main()
