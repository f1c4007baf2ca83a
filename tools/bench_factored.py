"""Cost of a factored (multi-discrete) action space (torchbeast_b200.action_space).  Prints the card and its power
limit, then:

1. the fused loss launch alone, tb_impala_loss_factored_f32 against tb_impala_loss_f32 at the same logit width
   (A = 8 as (3, 3, 2) and flat, A = 18 as (3, 3, 2, 2, 2, 2, 2, 2) and flat), as CUDA graphs of 50 launches, at
   T = 80, B = 32 and T = 80, B = 512.  Algorithmic bytes per launch: both logit tensors read once and the gradient
   written, (12 A + 8 D + 24) T B + 4 B (actions are D int64 per row; rewards, done, values read; five [T, B] outputs
   and grad_values written), against the H100 SXM's 3.35 TB/s.
2. the graphed monobeast.learn step (AtariNet + LSTM, T = 80, B = 32), flat A = 6 against (3, 3, 2), in alternating
   rounds.  The widths differ (6 against 8 logits): the step's difference includes the two extra policy rows.

    python tools/bench_factored.py [--rounds 3] [--steps 50]
"""
import argparse
import ctypes
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_legal_actions import time_legs  # noqa: E402
from tools.bench_trust_region import card, time_graph  # noqa: E402
from torchbeast_b200 import _lib, action_space, monobeast, optim  # noqa: E402

LAUNCHES = 50
PEAK = 3.35e12


def loss_bytes(T, B, A, D):
    return (12 * A + 8 * D + 24) * T * B + 4 * B


def loss_graph(T, B, dims):
    """A graph of LAUNCHES loss calls: the factored kernel, or for one component the flat one at that width."""
    A = sum(dims)
    rs = np.random.RandomState(T + B + A)
    cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
    f32 = np.float32
    tl = cu((1.5 * rs.randn(T, B, A)).astype(f32))
    bl = cu((1.5 * rs.randn(T, B, A)).astype(f32))
    acts = cu(np.stack([rs.randint(0, a, size=(T, B)) for a in dims], -1).astype(np.int64))
    rw, vals, bs = cu(rs.randn(T, B).astype(f32)), cu(rs.randn(T, B).astype(f32)), cu(rs.randn(B).astype(f32))
    done = cu(rs.rand(T, B) < 0.05)
    outs = [torch.empty(T, B, device="cuda") for _ in range(5)]
    losses = torch.empty(4, device="cuda")
    gl, gv = torch.empty(T + 1, B, A, device="cuda"), torch.empty(T + 1, B, device="cuda")
    ws = _lib.workspace()
    p = _lib.ptr
    space = action_space.c_space(dims) if len(dims) > 1 else None
    act = acts if space is not None else acts[..., 0].contiguous()

    def call():
        args = (p(bl), p(tl), p(act), p(rw), p(done), None, p(vals), p(bs), T, B, A, 0.99, 0.5, 0.01, 1, 1.0, 1.0,
                None, None, None, None, None, 0, None, None, None, None, *[p(o) for o in outs], p(losses), p(gl),
                p(gv), 1)
        if space is None:
            _lib.check(_lib.lib().tb_impala_loss_f32(*args, p(ws), _lib.stream_ptr()), "tb_impala_loss_f32")
        else:
            _lib.check(_lib.lib().tb_impala_loss_factored_f32(*args, ctypes.byref(space), p(ws), _lib.stream_ptr()),
                       "tb_impala_loss_factored_f32")
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            call()
    return g, (tl, bl, acts, act, rw, vals, bs, done, outs, losses, gl, gv)


def learn_step(num_actions):
    T, B = 80, 32
    model = monobeast.AtariNet((4, 84, 84), num_actions, True)
    actor = monobeast.AtariNet((4, 84, 84), num_actions, True)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5,
                                  entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=True)
    dims = action_space.dims_of(num_actions) or (num_actions,)
    g = torch.Generator().manual_seed(2)
    act = torch.stack([torch.randint(0, a, (T + 1, B), generator=g) for a in dims], -1)
    if action_space.dims_of(num_actions) is None:
        act = act[..., 0]
    batch = dict(frame=torch.randint(0, 255, (T + 1, B, 4, 84, 84), generator=g, dtype=torch.uint8),
                 reward=torch.randn(T + 1, B, generator=g), done=torch.rand(T + 1, B, generator=g) < 0.05,
                 episode_return=torch.randn(T + 1, B, generator=g),
                 policy_logits=torch.randn(T + 1, B, sum(dims), generator=g), action=act, last_action=act.clone())
    batch = {k: v.cuda() for k, v in batch.items()}
    state = model.initial_state(B)
    return lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_factored needs a GPU")
    print("card: %s" % card())
    print("\n1. fused loss launch alone, graphs of %d launches (median of %d rounds, per launch)"
          % (LAUNCHES, args.rounds))
    print("%-34s %10s %10s %10s %8s" % ("T, B, space", "us", "MB", "GB/s", "of peak"))
    for T, B in ((80, 32), (80, 512)):
        for factored, flat in (((3, 3, 2), (8,)), ((3, 3, 2, 2, 2, 2, 2, 2), (18,))):
            legs = {}
            for dims in (flat, factored):
                g, keep = loss_graph(T, B, dims)
                legs[dims] = (g, keep)
            us = {dims: [] for dims in legs}
            for _ in range(args.rounds):       # alternate the two kernels round by round
                for dims, (g, _k) in legs.items():
                    us[dims].append(time_graph(g) / LAUNCHES * 1e3)
            for dims, xs in us.items():
                m = statistics.median(xs)
                nb = loss_bytes(T, B, sum(dims), len(dims))
                name = "%d, %d, %s" % (T, B, "flat A=%d" % dims[0] if len(dims) == 1 else str(dims))
                print("%-34s %10.2f %10.3f %10.1f %7.1f%%   (rounds %s)" % (
                    name, m, nb * 1e-6, nb / m * 1e-3, 100 * nb / (m * 1e-6) / PEAK, ", ".join("%.2f" % x for x in xs)))
    print("\n2. graphed learn step, AtariNet + LSTM, T=80, B=32, ms per step")
    res = time_legs({"flat A=6": learn_step(6), "(3, 3, 2)": learn_step((3, 3, 2))}, args.rounds, args.steps)
    for name, xs in res.items():
        print("%-12s median %.3f ms  rounds %s" % (name, statistics.median(xs), ", ".join("%.3f" % x for x in xs)))


if __name__ == "__main__":
    main()
