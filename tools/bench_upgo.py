"""Cost of UPGO (flags.upgo_cost).  Prints the card and its power limit, then:

1. the UPGO launch alone (tb_upgo_loss_f32, after one loss launch has written log_rhos, the losses and grad_logits), as
   a CUDA graph of 50 launches, at T=80,B=32, T=600,B=128 and T=20,B=8192 with A=6.  Algorithmic bytes per launch:
   (12A + 25)*T*B + 4*B + 16 (target logits, actions, rewards, bool done, values, log_rhos and upgo_adv once each,
   grad_logits read and written, the bootstrap, the cost, the loss and the total).
2. the graphed monobeast.learn step (AtariNet + LSTM, T=80, B=32) with UPGO off and on, in alternating rounds.

    python tools/bench_upgo.py [--rounds 3] [--steps 50]
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

A = 6
LAUNCHES = 50


def upgo_bytes(T, B):
    return (12 * A + 25) * T * B + 4 * B + 16


def upgo_graph(T, B):
    """A graph of LAUNCHES tb_upgo_loss_f32 calls on the outputs of one loss launch (each adds into grad_logits)."""
    rs = np.random.RandomState(T + B)
    cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
    tl = cu((1.5 * rs.randn(T, B, A)).astype(np.float32))
    act, rw = cu(rs.randint(0, A, size=(T, B))), cu(rs.randn(T, B).astype(np.float32))
    done, vals = cu(rs.rand(T, B) < 0.05), cu(rs.randn(T, B).astype(np.float32))
    bs = cu(rs.randn(B).astype(np.float32))
    loss = learner.impala_loss_fwd_bwd(cu((1.5 * rs.randn(T, B, A)).astype(np.float32)), tl, act, rw, done, vals, bs)
    cost, adv, out = torch.ones(1, device="cuda"), torch.empty(T, B, device="cuda"), torch.empty(1, device="cuda")
    p = _lib.ptr

    def call():
        _lib.check(_lib.lib().tb_upgo_loss_f32(
            p(tl), p(act), p(rw), p(done.view(torch.uint8)), None, p(vals), p(bs), T, B, A, 0.99, 1, 1.0, None, None,
            None, None, None, 0, p(loss.log_rhos), None, None, p(cost), p(adv), p(out), p(loss.losses),
            p(loss.grad_logits), p(_lib.workspace()), _lib.stream_ptr()), "tb_upgo_loss_f32")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()   # the stream's workspace outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            call()
    return g, (tl, act, rw, done, vals, bs, loss, cost, adv, out)


def learn_step(upgo):
    T, B = 80, 32
    model = monobeast.AtariNet((4, 84, 84), A, True)
    actor = monobeast.AtariNet((4, 84, 84), A, True)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5,
                                  entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=True,
                                  upgo_cost=1.0 if upgo else None)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=2).items()}
    state = model.initial_state(B)
    return lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_upgo needs a GPU")
    print("card: %s" % card())
    print("\n1. UPGO launch alone, graphs of %d launches, A = %d (median of %d rounds, per launch)" % (
        LAUNCHES, A, args.rounds))
    print("%-16s %12s %12s %12s" % ("T, B", "us", "MB", "GB/s"))
    for T, B in ((80, 32), (600, 128), (20, 8192)):
        g, _keep = upgo_graph(T, B)
        us = [time_graph(g) / LAUNCHES * 1e3 for _ in range(args.rounds)]
        m = statistics.median(us)
        print("%-16s %12.2f %12.3f %12.1f   (rounds %s)" % ("%d, %d" % (T, B), m, upgo_bytes(T, B) * 1e-6,
                                                           upgo_bytes(T, B) / m * 1e-3, ", ".join("%.2f" % x for x in us)))
    print("\n2. graphed learn step, AtariNet + LSTM, T=80, B=32, ms per step")
    legs = {"off": learn_step(False), "on (cost 1.0)": learn_step(True)}
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
        print("%-16s median %.3f ms  rounds %s" % (name, statistics.median(xs), ", ".join("%.3f" % x for x in xs)))


if __name__ == "__main__":
    main()
