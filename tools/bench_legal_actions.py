"""Cost of legal-action masks (a legal_actions leaf, torchbeast_b200.legal_actions).  Prints the card and its power
limit, then:

1. the masking launch alone (tb_mask_logits_f32 with the action check), as a CUDA graph of 50 launches, at
   (T+1)*B rows of A actions = 81*32*6, 601*128*6, 81*32*18 and 81*32*362.  Algorithmic bytes per launch:
   N*A*(4 + 4 + 1) + 8*N (logits read and written, the mask read, the actions read), and the share of the H100 SXM's
   3.35 TB/s.
2. the graphed monobeast.learn step (AtariNet + LSTM, T=80, B=32) with no leaf, an all-legal leaf and a random mask,
   in alternating rounds.
3. the graphed T=1 acting call (AtariNet + LSTM, GraphedActor with a sampler) at B = 1, 48 and 512, with and without
   the mask, in alternating rounds.

    python tools/bench_legal_actions.py [--rounds 3] [--steps 50]
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
from torchbeast_b200 import _lib, monobeast, optim  # noqa: E402
from torchbeast_b200.acting import GraphedActor  # noqa: E402
from torchbeast_b200.legal_actions import MASKED_LOGIT  # noqa: E402
from torchbeast_b200.sampling import ActionSampler  # noqa: E402

LAUNCHES = 50
PEAK = 3.35e12


def mask_bytes(N, A):
    return N * A * (4 + 4 + 1) + 8 * N


def random_mask(shape, seed):
    """About half the actions legal, and at least one per row."""
    rs = np.random.RandomState(seed)
    legal = rs.rand(*shape) < 0.5
    rows = legal.reshape(-1, shape[-1])
    rows[np.arange(rows.shape[0]), rs.randint(0, shape[-1], rows.shape[0])] = True
    return legal


def mask_graph(N, A):
    """A graph of LAUNCHES out-of-place tb_mask_logits_f32 calls with the action check."""
    rs = np.random.RandomState(N + A)
    legal = random_mask((N, A), N + A)
    actions = np.array([rs.choice(np.flatnonzero(r)) for r in legal], np.int64)
    cu = lambda x: torch.from_numpy(x).cuda()   # noqa: E731
    x, lg, act = cu((2 * rs.randn(N, A)).astype(np.float32)), cu(legal.astype(np.uint8)), cu(actions)
    out = torch.empty_like(x)
    p = _lib.ptr

    def call():
        _lib.check(_lib.lib().tb_mask_logits_f32(p(x), p(out), p(lg), p(act), N, A, MASKED_LOGIT, _lib.stream_ptr()),
                   "tb_mask_logits_f32")
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            call()
    return g, (x, lg, act, out)


def learn_step(leaf):
    """leaf: None, "all" (every action legal) or "random"."""
    T, B, A = 80, 32, 6
    model = monobeast.AtariNet((4, 84, 84), A, True)
    actor = monobeast.AtariNet((4, 84, 84), A, True)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5,
                                  entropy_cost=0.0006, grad_norm_clipping=40.0, cuda_graph=True)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=2).items()}
    if leaf is not None:
        legal = np.ones((T + 1, B, A), bool) if leaf == "all" else random_mask((T + 1, B, A), 3)
        rs = np.random.RandomState(4)
        acts = np.array([rs.choice(np.flatnonzero(r)) for r in legal.reshape(-1, A)], np.int64).reshape(T + 1, B)
        batch["legal_actions"] = torch.from_numpy(legal).cuda()
        batch["action"][1:] = torch.from_numpy(acts[:-1]).cuda()   # action t+1 was chosen at frame t
    state = model.initial_state(B)
    return lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)


def acting_call(B, masked):
    A = 6
    model = monobeast.AtariNet((4, 84, 84), A, True)
    model.reset_parameters_like_torch(seed=5)
    model.action_sampler = ActionSampler(6)
    batch = LT.synthetic_batch(0, B, A, seed=7)
    inputs = {k: batch[k].cuda() for k in ("frame", "reward", "done", "last_action")}
    if masked:
        inputs["legal_actions"] = torch.from_numpy(random_mask((1, B, A), 8)).cuda()
    state = model.initial_state(B)
    actor = GraphedActor(model)
    return lambda: actor(inputs, state)


def time_legs(legs, rounds, steps):
    for step in legs.values():
        for _ in range(5):
            step()
    torch.cuda.synchronize()
    res = {k: [] for k in legs}
    for _ in range(rounds):
        for name, step in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                step()
            torch.cuda.synchronize()
            res[name].append((time.perf_counter() - t0) / steps * 1e3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_legal_actions needs a GPU")
    print("card: %s" % card())
    print("\n1. masking launch alone (with the action check), graphs of %d launches (median of %d rounds, per launch)"
          % (LAUNCHES, args.rounds))
    print("%-16s %10s %10s %10s %8s" % ("N, A", "us", "MB", "GB/s", "of peak"))
    for N, A in ((81 * 32, 6), (601 * 128, 6), (81 * 32, 18), (81 * 32, 362)):
        g, _keep = mask_graph(N, A)
        us = [time_graph(g) / LAUNCHES * 1e3 for _ in range(args.rounds)]
        m = statistics.median(us)
        nb = mask_bytes(N, A)
        print("%-16s %10.2f %10.3f %10.1f %7.1f%%   (rounds %s)" % (
            "%d, %d" % (N, A), m, nb * 1e-6, nb / m * 1e-3, 100 * nb / (m * 1e-6) / PEAK,
            ", ".join("%.2f" % x for x in us)))
    print("\n2. graphed learn step, AtariNet + LSTM, T=80, B=32, ms per step")
    res = time_legs({"no leaf": learn_step(None), "all-legal leaf": learn_step("all"),
                     "random mask": learn_step("random")}, args.rounds, args.steps)
    for name, xs in res.items():
        print("%-20s median %.3f ms  rounds %s" % (name, statistics.median(xs), ", ".join("%.3f" % x for x in xs)))
    print("\n3. graphed T=1 acting call, AtariNet + LSTM with a sampler, ms per call")
    for B in (1, 48, 512):
        res = time_legs({"no mask": acting_call(B, False), "mask": acting_call(B, True)}, args.rounds, 4 * args.steps)
        print("B=%-4d %s" % (B, "   ".join("%s median %.4f ms (rounds %s)" % (
            name, statistics.median(xs), ", ".join("%.4f" % x for x in xs)) for name, xs in res.items())))


if __name__ == "__main__":
    main()
