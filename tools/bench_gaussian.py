"""Cost of a continuous (diagonal-Gaussian) action space (torchbeast_b200.action_space.Gaussian).  Prints the card and
its power limit, then:

1. the fused loss launch alone, tb_impala_loss_gaussian_f32 against tb_impala_loss_f32 at the same row width A = 2D
   (D = 6: A = 12; D = 21: A = 42), as CUDA graphs of 50 launches, at T = 80, B = 32 and T = 80, B = 512.
   Algorithmic bytes per Gaussian launch: both row tensors read once and the gradient written, (12 A + 4 D + 24) T B
   + 4 B (actions are D float32 per row; rewards, done, values read; five [T, B] outputs and grad_values written),
   against the H100 SXM's 3.35 TB/s.
2. the Gaussian sampler at acting sizes (T = 1, B = 1, 48, 512; D = 6), graphs of 50 launches reading (seed, step)
   from the device, against the categorical sampler at A = 12.
3. the graphed monobeast.learn step (AtariNet + LSTM, T = 80, B = 32), Gaussian(6) against flat A = 12, in
   alternating rounds.  Both policy layers are 12 wide; the Gaussian core is 6 columns narrower (519 against 525).

    python tools/bench_gaussian.py [--rounds 3] [--steps 50]
"""
import argparse
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_legal_actions import time_legs  # noqa: E402
from tools.bench_trust_region import card, time_graph  # noqa: E402
from torchbeast_b200 import _lib, monobeast, optim, sampling  # noqa: E402
from torchbeast_b200.action_space import Gaussian  # noqa: E402

LAUNCHES = 50
PEAK = 3.35e12


def loss_bytes(T, B, A, D):
    return (12 * A + (4 * D if D else 8) + 24) * T * B + 4 * B


def loss_graph(T, B, A, gaussian):
    """A graph of LAUNCHES loss calls at row width A: the Gaussian kernel (D = A / 2), or the flat one."""
    D = A // 2
    rs = np.random.RandomState(T + B + A)
    cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
    f32 = np.float32
    bl = np.concatenate([rs.randn(T, B, D), rs.uniform(-1, 0.5, (T, B, D))], -1).astype(f32)
    tl = cu((bl + 0.1 * rs.randn(T, B, A)).astype(f32))
    bl = cu(bl)
    if gaussian:
        act = cu(rs.randn(T, B, D).astype(f32))
    else:
        act = cu(rs.randint(0, A, size=(T, B)).astype(np.int64))
    rw, vals, bs = cu(rs.randn(T, B).astype(f32)), cu(rs.randn(T, B).astype(f32)), cu(rs.randn(B).astype(f32))
    done = cu(rs.rand(T, B) < 0.05)
    outs = [torch.empty(T, B, device="cuda") for _ in range(5)]
    losses = torch.empty(4, device="cuda")
    gl, gv = torch.empty(T + 1, B, A, device="cuda"), torch.empty(T + 1, B, device="cuda")
    ws = _lib.workspace()
    p = _lib.ptr
    fn = _lib.lib().tb_impala_loss_gaussian_f32 if gaussian else _lib.lib().tb_impala_loss_f32

    def call():
        _lib.check(fn(p(bl), p(tl), p(act), p(rw), p(done), None, p(vals), p(bs), T, B, A, 0.99, 0.5, 0.01, 1, 1.0,
                      1.0, None, None, None, None, None, 0, None, None, None, None, *[p(o) for o in outs], p(losses),
                      p(gl), p(gv), 1, p(ws), _lib.stream_ptr()), "impala loss")
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            call()
    return g, (tl, bl, act, rw, vals, bs, done, outs, losses, gl, gv)


def sampler_graph(B, D, gaussian):
    rows = torch.randn(1, B, 2 * D, device="cuda")
    seed_step = torch.tensor([7, 0], dtype=torch.int64, device="cuda")
    out = torch.empty(1, B, dtype=torch.int64, device="cuda")

    def call():
        if gaussian:
            return sampling.sample_gaussian(rows, D, None, seed_step=seed_step)
        _lib.check(_lib.lib().tb_sample_actions_dev_f32(_lib.ptr(rows), 1, B, 2 * D, _lib.ptr(seed_step), None,
                                                        _lib.ptr(out), _lib.stream_ptr()), "tb_sample_actions_dev_f32")
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            call()
    return g, (rows, seed_step, out)


def learn_step(num_actions):
    T, B = 80, 32
    model = monobeast.AtariNet((4, 84, 84), num_actions, True)
    actor = monobeast.AtariNet((4, 84, 84), num_actions, True)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5,
                                  entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=True)
    g = torch.Generator().manual_seed(2)
    if isinstance(num_actions, Gaussian):
        D = num_actions.dim
        act = torch.randn(T + 1, B, D, generator=g)
        logits = torch.cat([torch.randn(T + 1, B, D, generator=g), torch.full((T + 1, B, D), -0.5)], -1)
    else:
        act = torch.randint(0, num_actions, (T + 1, B), generator=g)
        logits = torch.randn(T + 1, B, num_actions, generator=g)
    batch = dict(frame=torch.randint(0, 255, (T + 1, B, 4, 84, 84), generator=g, dtype=torch.uint8),
                 reward=torch.randn(T + 1, B, generator=g), done=torch.rand(T + 1, B, generator=g) < 0.05,
                 episode_return=torch.randn(T + 1, B, generator=g), policy_logits=logits, action=act,
                 last_action=act.clone())
    batch = {k: v.cuda() for k, v in batch.items()}
    state = model.initial_state(B)
    return lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gaussian needs a GPU")
    print("card: %s" % card())
    print("\n1. fused loss launch alone, graphs of %d launches (median of %d rounds, per launch)"
          % (LAUNCHES, args.rounds))
    print("%-30s %10s %10s %10s %8s" % ("T, B, row", "us", "MB", "GB/s", "of peak"))
    for T, B in ((80, 32), (80, 512)):
        for A in (12, 42):
            legs = {kind: loss_graph(T, B, A, kind == "gaussian") for kind in ("flat", "gaussian")}
            us = {kind: [] for kind in legs}
            for _ in range(args.rounds):       # alternate the two kernels round by round
                for kind, (g, _k) in legs.items():
                    us[kind].append(time_graph(g) / LAUNCHES * 1e3)
            for kind, xs in us.items():
                m = statistics.median(xs)
                nb = loss_bytes(T, B, A, A // 2 if kind == "gaussian" else 0)
                name = "%d, %d, %s A=%d" % (T, B, kind, A)
                print("%-30s %10.2f %10.3f %10.1f %7.1f%%   (rounds %s)" % (
                    name, m, nb * 1e-6, nb / m * 1e-3, 100 * nb / (m * 1e-6) / PEAK, ", ".join("%.2f" % x for x in xs)))
    print("\n2. sampler at acting sizes, T=1, D=6 (A=12), graphs of %d launches, us per launch" % LAUNCHES)
    for B in (1, 48, 512):
        legs = {kind: sampler_graph(B, 6, kind == "gaussian") for kind in ("categorical", "gaussian")}
        us = {kind: [] for kind in legs}
        for _ in range(args.rounds):
            for kind, (g, _k) in legs.items():
                us[kind].append(time_graph(g) / LAUNCHES * 1e3)
        for kind, xs in us.items():
            print("B=%-4d %-12s median %.2f us  rounds %s" % (B, kind, statistics.median(xs),
                                                             ", ".join("%.2f" % x for x in xs)))
    print("\n3. graphed learn step, AtariNet + LSTM, T=80, B=32, ms per step")
    res = time_legs({"flat A=12": learn_step(12), "Gaussian(6)": learn_step(Gaussian(6))}, args.rounds, args.steps)
    for name, xs in res.items():
        print("%-12s median %.3f ms  rounds %s" % (name, statistics.median(xs), ", ".join("%.3f" % x for x in xs)))


if __name__ == "__main__":
    main()
