"""Ingest cost of stacked vs unstacked rollouts on one GPU, the two formats measured in alternating rounds.

    python tools/bench_ingest.py [--T 80] [--B 32] [--rounds 3] [--steps 30] [--actors 48] [--seconds 10]

Per format and round it reports:
  * h2d_mb / h2d_ms: bytes of one rollout slot (staging.spec_for) and the time of its host-to-device copy from pinned
    memory (CUDA events around `--steps` copies on the stager's copy stream);
  * learn_ms: monobeast.learn (AtariNet + LSTM, default backend, flags.cuda_graph) on a pinned host batch, per step, host
    clock around `--steps` steps that each read their stats back;
  * actors_fps: frames/s of `--actors` SyntheticActors threads -> RolloutStager -> two polybeast_learner.learn threads
    (the bench.py configs[2] pipeline) over `--seconds` seconds after a warm-up.
The card's name and power limit are printed first: the numbers belong to them.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import frames_np as F  # noqa: E402
from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import actors, monobeast, optim, polybeast_learner, staging  # noqa: E402

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (torch.cuda.get_device_name(0), q)


def h2d(fmt, T, B, A, steps):
    stager = staging.RolloutStager(staging.spec_for(T, B, A, use_last_action=False, frame_format=fmt), "cuda:0", depth=2)
    for _ in range(3):
        stager.put({})
        stager.release(stager.get()[1])
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stager._stream)
    for _ in range(steps):  # an empty put submits a whole slot; with two slots the next copy is queued behind this one
        stager.put({})
        stager.release(stager.get()[1])
    end.record(stager._stream)
    torch.cuda.synchronize()
    return stager.h2d_bytes / 1e6, start.elapsed_time(end) / steps


def learn(fmt, T, B, A, steps):
    stacks, done = F.simulate(T + 1, B, seed=1, done_prob=0.01)
    host = LT.synthetic_batch(T, B, A, seed=2)
    host["done"] = torch.from_numpy(done)
    host["frame"] = torch.from_numpy(stacks if fmt == "stacked" else F.unstack(stacks))
    host = {k: v.pin_memory() for k, v in host.items()}
    model = monobeast.AtariNet((4, 84, 84), A, True)
    actor = monobeast.AtariNet((4, 84, 84), A, True)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(unroll_length=T, batch_size=B, cuda_graph=True, **FLAGS)
    state = tuple(torch.zeros(2, B, 512 + A + 1).pin_memory() for _ in range(2))
    for _ in range(3):
        monobeast.learn(flags, actor, model, host, state, opt, None)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        monobeast.learn(flags, actor, model, host, state, opt, None)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def pipeline(fmt, T, B, A, num_actors, seconds):
    model = monobeast.AtariNet((4, 84, 84), A, True)
    actor = monobeast.AtariNet((4, 84, 84), A, True)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    stager = staging.RolloutStager(staging.spec_for(T, B, A, use_last_action=False, frame_format=fmt), "cuda:0", depth=4)
    model._tb_stager = stager
    q = actors.LearnerQueue()
    pool = actors.SyntheticActors(stager, num_actors, T, B, A, q, state_shape=(2, 512 + A + 1), frame_format=fmt)
    flags = types.SimpleNamespace(unroll_length=T, batch_size=B, cuda_graph=True, **FLAGS)
    steps, marks = [0], {}

    class Log:
        def log(self, s):
            steps[0] += 1
            if steps[0] == 5:
                marks["t0"] = time.perf_counter()
            if "t0" in marks and "t1" not in marks and time.perf_counter() - marks["t0"] >= seconds:
                marks["t1"], marks["n"] = time.perf_counter(), steps[0] - 5
                pool.stop()

    lock = threading.Lock()
    pool.start()
    ths = [threading.Thread(target=polybeast_learner.learn, args=(flags, q, model, actor, opt, None, {}, Log(), lock))
           for _ in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    torch.cuda.synchronize()
    return marks["n"] * T * B / (marks["t1"] - marks["t0"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=80)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--A", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--actors", type=int, default=48)
    ap.add_argument("--seconds", type=float, default=10.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ingest measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    print("card: %s" % card(), flush=True)
    for r in range(args.rounds):
        for fmt in ("stacked", "unstacked"):
            mb, ms = h2d(fmt, args.T, args.B, args.A, args.steps)
            res = dict(round=r, format=fmt, h2d_mb=round(mb, 3), h2d_ms=round(ms, 3),
                       learn_ms=round(learn(fmt, args.T, args.B, args.A, args.steps), 3))
            if args.actors:
                res["actors_fps"] = round(pipeline(fmt, args.T, args.B, args.A, args.actors, args.seconds))
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
