"""Cost of the V-trace trust region (flags.trust_region_kl).  Prints the card and its power limit, then:

1. the fused loss kernel alone, without and with the trust region (beta at the median KL, so about half the rows are
   untrusted), each as a CUDA graph of 50 launches, at T=80,B=32, T=600,B=128 and T=20,B=8192.  Achieved bytes/s use
   the algorithmic bytes of the fused loss in BASELINE.md section 3, (12A+32)*T*B + 4*B + 12, plus 4*T*B for the KL
   output.
2. the graphed monobeast.learn step (AtariNet + LSTM, T=80, 16 fresh + 16 replayed columns) without and with the trust
   region, in alternating rounds.

    python tools/bench_trust_region.py [--rounds 3] [--steps 50]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import learner, monobeast, optim  # noqa: E402
from torchbeast_b200.replay import ReplayBuffer  # noqa: E402

A = 6


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def loss_bytes(T, B, trust):
    return (12 * A + 32) * T * B + 4 * B + 12 + (4 * T * B if trust else 0)


def loss_graph(T, B, beta, launches=50):
    rs = np.random.RandomState(T + B)
    cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
    tl = (1.5 * rs.randn(T, B, A)).astype(np.float32)
    kw = dict(behavior_policy_logits=cu((tl + 0.7 * rs.randn(T, B, A)).astype(np.float32)),
              target_policy_logits=cu(tl), actions=cu(rs.randint(0, A, size=(T, B))),
              rewards=cu(rs.randn(T, B).astype(np.float32)), done=cu(rs.rand(T, B) < 0.05),
              values=cu(rs.randn(T, B).astype(np.float32)), bootstrap_value=cu(rs.randn(B).astype(np.float32)))
    trust = None if beta is None else torch.full((1,), beta, dtype=torch.float32, device="cuda")
    call = lambda: learner.impala_loss_fwd_bwd(**kw, trust_region=trust)   # noqa: E731
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()   # allocations and the stream's workspace outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            call()
    return g, kw


def time_graph(g, reps=20):
    g.replay()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        g.replay()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / reps   # ms per graph


def learn_step(trust):
    T, Bf, R = 80, 16, 16
    model = monobeast.AtariNet((4, 84, 84), A, True)
    actor = monobeast.AtariNet((4, 84, 84), A, True)
    model.reset_parameters_like_torch(seed=1)
    model.replay = ReplayBuffer(256, R, seed=3, min_size=Bf)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5,
                                  entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=True,
                                  trust_region_kl=0.05 if trust else None)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, Bf, A, seed=2).items()}
    state = model.initial_state(Bf)
    return lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_trust_region needs a GPU")
    print("card: %s" % card())
    print("\n1. fused loss kernel, graphs of 50 launches (median of %d rounds, per launch)" % args.rounds)
    print("%-16s %12s %12s %12s %12s" % ("T, B", "off us", "on us", "off GB/s", "on GB/s"))
    for T, B in ((80, 32), (600, 128), (20, 8192)):
        g_off, kw = loss_graph(T, B, None)
        kl = learner.impala_loss_fwd_bwd(**kw, trust_region=np.inf)[1].kl
        beta = float(kl.median())
        g_on, _ = loss_graph(T, B, beta)
        off, on = [], []
        for _ in range(args.rounds):
            off.append(time_graph(g_off) / 50 * 1e3)
            on.append(time_graph(g_on) / 50 * 1e3)
        mo, mn = statistics.median(off), statistics.median(on)
        print("%-16s %12.2f %12.2f %12.1f %12.1f   (rounds off %s, on %s)" % (
            "%d, %d" % (T, B), mo, mn, loss_bytes(T, B, False) / mo * 1e-3, loss_bytes(T, B, True) / mn * 1e-3,
            ", ".join("%.2f" % x for x in off), ", ".join("%.2f" % x for x in on)))
    print("\n2. graphed learn step, T=80, 16 fresh + 16 replayed columns, ms per step")
    legs = {"off": learn_step(False), "on (beta=0.05)": learn_step(True)}
    for step in legs.values():
        for _ in range(5):
            step()
    torch.cuda.synchronize()
    res = {k: [] for k in legs}
    for r in range(args.rounds):
        for name, step in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
            res[name].append((time.perf_counter() - t0) / args.steps * 1e3)
    for name, xs in res.items():
        print("%-16s median %.3f ms  rounds %s" % (name, statistics.median(xs), ", ".join("%.3f" % x for x in xs)))


if __name__ == "__main__":
    main()
