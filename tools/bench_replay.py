"""Cost of experience replay in the learner step, measured in alternating rounds.

    python tools/bench_replay.py [--rounds 3] [--steps 50] [--T 80] [--capacity 512]

Reports, after the card's name and power limit (the numbers belong to them):
  * learn_ms: the graphed monobeast.learn step (AtariNet + LSTM, default backend, RMSprop, device-resident batch, stats
    read back every step) at learner batch width 32, for (Bf, R) = (32, 0) (no buffer), (16, 16) and (24, 8), with
    stacked and with unstacked frames; CUDA events around `--steps` steps after the captures and a warm-up, the six
    configurations in a different order each round;
  * mix_us / GB/s: tb_replay_mix alone, 50 launches captured in a CUDA graph and replayed, with the achieved rate of
    the algorithmic bytes, sum over leaves of outer * row_bytes * (3*Bf + 2*R), against 3.35 TB/s.
Writes nothing.
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
from torchbeast_b200 import _lib, monobeast, optim  # noqa: E402
from torchbeast_b200.replay import ReplayBuffer, _Leaf  # noqa: E402

FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)
A = 6
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (torch.cuda.get_device_name(0), q)


def make_batch(T, B, frames, seed):
    b = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=seed).items()}
    if frames == "unstacked":
        b["frame"] = torch.randint(0, 256, (T + 4, B, 84, 84), dtype=torch.uint8, device="cuda")
    return b


class Setup:
    def __init__(self, T, Bf, R, frames, capacity):
        self.model = monobeast.AtariNet((4, 84, 84), A, True)
        self.actor = monobeast.AtariNet((4, 84, 84), A, True)
        self.model.reset_parameters_like_torch(seed=1)
        self.actor.copy_params_from(self.model)
        if R:
            self.model.replay = ReplayBuffer(capacity, R, seed=7)
        self.opt = optim.RMSprop(self.model, lr=0.00048, momentum=0, eps=0.01, alpha=0.99)
        self.flags = types.SimpleNamespace(unroll_length=T, batch_size=Bf, cuda_graph=True, **FLAGS)
        self.batch = make_batch(T, Bf, frames, seed=2)
        self.state = tuple(torch.zeros(2, Bf, 512 + A + 1, device="cuda") for _ in range(2))
        for _ in range(3):   # captures (warm-up phase, then mixing phase) and the buffer past its warm-up
            self.learn()

    def learn(self):
        return monobeast.learn(self.flags, self.actor, self.model, self.batch, self.state, self.opt, None)


def learn_ms(setup, steps, warmup=5):
    for _ in range(warmup):
        setup.learn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        setup.learn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def mix_alone(T, Bf, R, frames, capacity, launches=50, replays=10):
    """(microseconds per tb_replay_mix, algorithmic bytes per call) on a full ring."""
    buf = ReplayBuffer(capacity, R, seed=3)
    batch = make_batch(T, Bf, frames, seed=4)
    state = tuple(torch.zeros(2, Bf, 512 + A + 1, device="cuda") for _ in range(2))
    while buf.size < capacity:
        buf.mix(batch, state)
    fresh = [t.contiguous() for _, t in buf._leaves(batch, state)]
    outs = [torch.empty((t.shape[0], Bf + R) + tuple(t.shape[2:]), dtype=t.dtype, device="cuda") for t in fresh]
    slots = torch.empty(R, dtype=torch.int64, device="cuda")
    rows = [(f.shape[0], f[0, 0].numel() * f.element_size()) for f in fresh]
    table = (_Leaf * len(fresh))(*[_Leaf(f.data_ptr(), o.data_ptr(), r.data_ptr(), outer, rb)
                                   for f, o, r, (outer, rb) in zip(fresh, outs, buf.rings, rows)])
    nbytes = sum(outer * rb * (3 * Bf + 2 * R) for outer, rb in rows)

    def call():
        _lib.check(_lib.lib().tb_replay_mix(table, len(fresh), Bf, R, capacity, _lib.ptr(buf.state[2:]),
                                            _lib.ptr(buf.state[:2]), 0, _lib.ptr(slots), _lib.stream_ptr()),
                   "tb_replay_mix")

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(launches):
            call()
    graph.replay()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(replays):
        graph.replay()
    end.record()
    torch.cuda.synchronize()
    return 1e3 * start.elapsed_time(end) / (launches * replays), nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=80)
    ap.add_argument("--capacity", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_replay measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    print("card: %s" % card(), flush=True)
    configs = [(bf, r, fr) for fr in ("stacked", "unstacked") for bf, r in ((32, 0), (16, 16), (24, 8))]
    for Bf, R, frames in configs:
        if R:
            us, nbytes = mix_alone(args.T, Bf, R, frames, args.capacity)
            print(json.dumps(dict(bench="tb_replay_mix", T=args.T, Bf=Bf, R=R, frames=frames, mix_us=round(us, 2),
                                  algorithmic_MB=round(nbytes / 1e6, 1), GB_per_s=round(nbytes / us / 1e3, 1),
                                  share_of_3_35_TB_per_s=round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3))), flush=True)
    setups = {c: Setup(args.T, c[0], c[1], c[2], args.capacity) for c in configs}
    times = {c: [] for c in configs}
    for r in range(args.rounds):
        order = configs if r % 2 == 0 else configs[::-1]
        for c in order:
            times[c].append(learn_ms(setups[c], args.steps))
    for c in configs:
        t = times[c]
        print(json.dumps(dict(bench="graphed learn", T=args.T, Bf=c[0], R=c[1], frames=c[2], learn_ms=[round(x, 3) for x in t],
                              median_ms=round(sorted(t)[len(t) // 2], 3),
                              spread_ms=round(max(t) - min(t), 3))), flush=True)


if __name__ == "__main__":
    main()
