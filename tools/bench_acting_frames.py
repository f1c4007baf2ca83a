"""Graphed acting call with stacked frames vs newest frames (torchbeast_b200.acting.FrameHistory).

    python tools/bench_acting_frames.py [--nets atari,resnet] [--reps 100] [--rounds 5] [--fill_reps 1000] [--cold_reps 200]

For AtariNet+LSTM and ResNet+LSTM (default precision, training mode with the seeded sampler) at B in {1, 48, 512}, one
GraphedActor call per environment step, started from pinned host tensors as an actor's step arrives: the frame leaf
u8 [1, B, 4, 84, 84] (stacked) or [1, B, 84, 84] (newest; the history rebuilds the stack on the GPU), reward, done and
last_action.  The host-to-device copies are therefore inside the timed window.  CUDA events around `--reps` calls back
to back, the two formats alternating over `--rounds` rounds, median round reported.  Also reported: the bytes the call
copies host-to-device, and the fill kernel's own time at T = 1, twice: L2-warm (CUDA events around `--fill_reps`
launches of tb_frame_history_fill_u8 on one set of buffers, replayed from a CUDA graph of 100 launches so that the
host's launch cost is left out) and L2-cold (the median of `--cold_reps` single launches, each after a 256 MB write that
evicts the L2, as an acting call meets the history).  The card's name and power limit are printed first.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

A = 6


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (torch.cuda.get_device_name(0), q)


def host_step(B, seed):
    """One acting step's leaves in pinned host memory, in both frame formats."""
    rs = np.random.RandomState(seed)
    stacked = rs.randint(0, 256, size=(1, B, 4, 84, 84), dtype=np.uint8)
    leaves = dict(reward=rs.randn(1, B).astype(np.float32), done=rs.rand(1, B) < 0.01,
                  last_action=rs.randint(0, A, size=(1, B)).astype(np.int64))
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
    common = {k: pin(v) for k, v in leaves.items()}
    return dict(common, frame=pin(stacked)), dict(common, frame=pin(stacked[:, :, 3]))


def timed(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def bench_net(net, sizes, reps, rounds, fill_reps, cold_reps):
    from torchbeast_b200 import monobeast, polybeast_learner
    from torchbeast_b200.acting import FrameHistory, GraphedActor
    from torchbeast_b200.sampling import ActionSampler
    model = polybeast_learner.Net(A, True) if net == "resnet" else monobeast.AtariNet((4, 84, 84), A, True)
    model.reset_parameters_like_torch(seed=0)
    model.train()
    model.action_sampler = ActionSampler(seed=0)
    model.frame_history = FrameHistory(max(sizes))
    actor = GraphedActor(model)
    for B in sizes:
        stacked, newest = host_step(B, seed=B)
        state = model.initial_state(B)
        calls = {"stacked": lambda: actor(stacked, state), "newest": lambda: actor(newest, state)}
        with torch.no_grad():
            for fn in calls.values():  # capture + warm-up
                for _ in range(5):
                    fn()
            times = {k: [] for k in calls}
            for _ in range(rounds):
                for k, fn in calls.items():
                    times[k].append(timed(fn, reps))
        frames = torch.zeros(4, B, 84, 84, dtype=torch.uint8, device="cuda")
        done = torch.zeros(1, B, dtype=torch.uint8, device="cuda")
        ids = torch.arange(B, dtype=torch.int64, device="cuda")
        # the kernel's own time: 100 launches captured in one graph, so the host's launch cost stays out of the window
        model.frame_history.fill(frames, done, ids)
        torch.cuda.synchronize()
        fills = torch.cuda.CUDAGraph()
        with torch.cuda.graph(fills):
            for _ in range(100):
                model.frame_history.fill(frames, done, ids)
        fills.replay()
        fill_us = float(np.median([timed(fills.replay, max(1, fill_reps // 100)) for _ in range(rounds)])) * 10
        # Those launches reuse one set of buffers that fits in L2.  Cold: before each launch a 256 MB write evicts the
        # L2 (50 MB), and events time the launch alone; the write is still running when the launch is enqueued, so no
        # host gap falls inside the window.
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        cold = []
        for _ in range(cold_reps):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            flush.fill_(1)
            start.record()
            model.frame_history.fill(frames, done, ids)
            end.record()
            cold.append((start, end))
        torch.cuda.synchronize()
        cold_us = float(np.median([s.elapsed_time(e) for s, e in cold])) * 1e3
        del flush
        print(json.dumps(dict(
            net=net, precision=model.precision, B=B,
            stacked_ms=round(float(np.median(times["stacked"])), 4), newest_ms=round(float(np.median(times["newest"])), 4),
            stacked_h2d_bytes=sum(v.numel() * v.element_size() for v in stacked.values()),
            newest_h2d_bytes=sum(v.numel() * v.element_size() for v in newest.values()),
            fill_kernel_us_l2_warm=round(fill_us, 2), fill_kernel_us_l2_cold=round(cold_us, 2),
            fill_bytes=B * 84 * 84 * 10,  # reads history (3) + newest frame (1), writes rows 0..2 (3) + history (3)
            rounds_ms=dict(stacked=[round(t, 4) for t in times["stacked"]], newest=[round(t, 4) for t in times["newest"]]))),
            flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="atari,resnet")
    ap.add_argument("--sizes", default="1,48,512")
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--fill_reps", type=int, default=1000)
    ap.add_argument("--cold_reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_acting_frames measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    print("card: %s" % card(), flush=True)
    print("timing: %d graphed calls per CUDA-event pair from pinned host leaves, median of %d alternating rounds"
          % (args.reps, args.rounds), flush=True)
    for net in args.nets.split(","):
        bench_net(net, [int(b) for b in args.sizes.split(",")], args.reps, args.rounds, args.fill_reps,
                  args.cold_reps)


if __name__ == "__main__":
    main()
