"""Cost of kickstarting (flags.kickstart_cost with model.teacher).  Prints the card and its power limit, then:

1. the kickstarting launch alone (tb_kickstart_loss_f32, adding into a grad_logits buffer), as a CUDA graph of 50
   launches, at (T, B, A) = (80, 32, 6), (600, 128, 6), (20, 8192, 6) and (80, 32, 23).  Algorithmic bytes per launch:
   16*A*T*B + 4*B + 12 (the two logits read, grad_logits read and written, the weights, the cost, the outputs), and
   the share of the H100 SXM's 3.35 TB/s.
2. the graphed monobeast.learn step (AtariNet + LSTM learner, T=80, B=32) with no teacher, a feed-forward AtariNet
   teacher and an AtariNet + LSTM teacher, in alternating rounds, and each teacher's workspace bytes.

    python tools/bench_kickstart.py [--rounds 3] [--steps 50]
"""
import argparse
import os
import statistics
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import learner_torch as LT  # noqa: E402
from tools.bench_trust_region import card, time_graph  # noqa: E402
from torchbeast_b200 import _lib, learner, monobeast, optim  # noqa: E402
from torchbeast_b200.kickstart import Teacher  # noqa: E402

LAUNCHES = 50
PEAK = 3.35e12


def kickstart_bytes(T, B, A):
    return 16 * A * T * B + 4 * B + 12


def kickstart_graph(T, B, A):
    """A graph of LAUNCHES weighted tb_kickstart_loss_f32 calls (each adds into grad_logits and the total)."""
    rs = np.random.RandomState(T + B + A)
    cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
    teacher, target = cu((2 * rs.randn(T, B, A)).astype(np.float32)), cu((2 * rs.randn(T, B, A)).astype(np.float32))
    w = cu(rs.rand(B).astype(np.float32))
    gl, losses = torch.zeros(T + 1, B, A, device="cuda"), torch.zeros(4, device="cuda")
    cost, out = torch.full((1,), 1e-3, device="cuda"), torch.empty(2, device="cuda")
    p = _lib.ptr

    def call():
        _lib.check(_lib.lib().tb_kickstart_loss_f32(p(teacher), p(target), T, B, A, p(w), p(cost), p(out), p(losses),
                                                    p(gl), p(_lib.workspace()), _lib.stream_ptr()),
                   "tb_kickstart_loss_f32")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()   # the stream's workspace outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            call()
    return g, (teacher, target, w, gl, losses, cost, out)


def learn_step(teacher):
    """teacher: None, "ff" or "lstm".  Returns (step, teacher workspace bytes)."""
    T, B, A = 80, 32, 6
    model = monobeast.AtariNet((4, 84, 84), A, True)
    actor = monobeast.AtariNet((4, 84, 84), A, True)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5,
                                  entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=True)
    if teacher is not None:
        net = monobeast.AtariNet((4, 84, 84), A, teacher == "lstm")
        net.reset_parameters_like_torch(seed=2)
        model.teacher = Teacher(net)
        flags.kickstart_cost = 1.0
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=2).items()}
    state = model.initial_state(B)
    step = lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)   # noqa: E731
    ws = 0 if teacher is None else int(_lib.lib().tb_atarinet_workspace_bytes(
        T + 1, B, A, int(teacher == "lstm"), monobeast.AtariNet.PRECISIONS[model.precision]))
    return step, ws


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_kickstart needs a GPU")
    print("card: %s" % card())
    print("\n1. kickstarting launch alone (weighted), graphs of %d launches (median of %d rounds, per launch)" % (
        LAUNCHES, args.rounds))
    print("%-16s %10s %10s %10s %8s" % ("T, B, A", "us", "MB", "GB/s", "of peak"))
    for T, B, A in ((80, 32, 6), (600, 128, 6), (20, 8192, 6), (80, 32, 23)):
        g, _keep = kickstart_graph(T, B, A)
        us = [time_graph(g) / LAUNCHES * 1e3 for _ in range(args.rounds)]
        m = statistics.median(us)
        nb = kickstart_bytes(T, B, A)
        print("%-16s %10.2f %10.3f %10.1f %7.1f%%   (rounds %s)" % (
            "%d, %d, %d" % (T, B, A), m, nb * 1e-6, nb / m * 1e-3, 100 * nb / (m * 1e-6) / PEAK,
            ", ".join("%.2f" % x for x in us)))
    print("\n2. graphed learn step, AtariNet + LSTM learner, T=80, B=32, ms per step")
    legs, wsb = {}, {}
    for name, t in (("no teacher", None), ("AtariNet teacher", "ff"), ("AtariNet+LSTM teacher", "lstm")):
        legs[name], wsb[name] = learn_step(t)
    for step in legs.values():
        for _ in range(5):
            step()
    torch.cuda.synchronize()
    res = {k: [] for k in legs}
    for _ in range(args.rounds):
        for name, step in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
            res[name].append((time.perf_counter() - t0) / args.steps * 1e3)
    for name, xs in res.items():
        print("%-24s median %.3f ms  rounds %s  teacher workspace %.1f MB" % (
            name, statistics.median(xs), ", ".join("%.3f" % x for x in xs), wsb[name] * 1e-6))


if __name__ == "__main__":
    main()
