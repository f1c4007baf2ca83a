"""Cost of MLPNet (vector observations, torchbeast_b200.nets.MLPNet).  Prints the card and its power limit, then:

1. the graphed monobeast.learn step at T = 80, O = 17, Gaussian(6), hidden (256, 256), with and without the LSTM, at
   B = 32 and B = 256, with and without observation normalisation, in alternating rounds (ms per step).
2. the staging kernel (tb_obs_stage, split-bf16 operand) and the two statistics kernels (tb_obs_norm_sums over rows
   1..T, tb_obs_norm_update) alone, as CUDA graphs of 50 launches, at T + 1 = 81, B = 256 and O = 17 / 376.
   Algorithmic bytes: staging reads 4 N O and writes 4 N ld (two bf16 planes, ld = O rounded up to 8) plus 16 O of
   statistics; the sums read 4 T B O and write 24 O; the update reads 48 O and writes 24 O.  Against 3.35 TB/s.
3. the graphed T = 1 acting call (acting.GraphedActor, sampler attached, LSTM net) at B = 1, 48 and 512.
4. for context, the same net and loss in plain torch (fp32, autograd, the oracle's V-trace from oracle/learner_torch,
   RMSprop), at flat A = 12, the same policy width: that V-trace is categorical.

    python tools/bench_mlpnet.py [--rounds 3] [--steps 30]
"""
import argparse
import os
import statistics
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from oracle import learner_torch as LT  # noqa: E402
from tools.bench_legal_actions import time_legs  # noqa: E402
from tools.bench_trust_region import card, time_graph  # noqa: E402
from torchbeast_b200 import _lib, monobeast, nets, optim  # noqa: E402
from torchbeast_b200.acting import GraphedActor  # noqa: E402
from torchbeast_b200.action_space import Gaussian  # noqa: E402
from torchbeast_b200.sampling import ActionSampler  # noqa: E402

LAUNCHES = 50
PEAK = 3.35e12
O, D, T, HIDDEN = 17, 6, 80, (256, 256)
FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006,
             grad_norm_clipping=40.0)


def batch_for(B, obs=O, gaussian=True, seed=2):
    g = torch.Generator().manual_seed(seed)
    if gaussian:
        act = torch.randn(T + 1, B, D, generator=g)
        logits = torch.cat([torch.randn(T + 1, B, D, generator=g), torch.full((T + 1, B, D), -0.5)], -1)
    else:
        act = torch.randint(0, 2 * D, (T + 1, B), generator=g)
        logits = torch.randn(T + 1, B, 2 * D, generator=g)
    b = dict(frame=torch.randn(T + 1, B, obs, generator=g) * 3 + 1, reward=torch.randn(T + 1, B, generator=g),
             done=torch.rand(T + 1, B, generator=g) < 0.05, episode_return=torch.randn(T + 1, B, generator=g),
             policy_logits=logits, action=act, last_action=act.clone())
    return {k: v.cuda() for k, v in b.items()}


def learn_step(B, use_lstm, norm):
    kw = dict(hidden=HIDDEN, use_lstm=use_lstm, normalize_observations=norm)
    model, actor = nets.MLPNet(O, Gaussian(D), **kw), nets.MLPNet(O, Gaussian(D), **kw)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(**FLAGS, cuda_graph=True)
    batch, state = batch_for(B), model.initial_state(B)
    return lambda: monobeast.learn(flags, actor, model, batch, state, opt, None)


def torch_step(B, use_lstm):
    """The same net (fp32 torch modules) and the IMPALA loss with the oracle's V-trace, autograd, RMSprop."""
    core = HIDDEN[-1] + 1 + 2 * D
    torso = torch.nn.Sequential(torch.nn.Linear(O, HIDDEN[0]), torch.nn.ReLU(), torch.nn.Linear(*HIDDEN),
                                torch.nn.ReLU()).cuda()
    lstm = torch.nn.LSTM(core, core, 2).cuda() if use_lstm else None
    policy, baseline = torch.nn.Linear(core, 2 * D).cuda(), torch.nn.Linear(core, 1).cuda()
    params = [p for m in (torso, lstm, policy, baseline) if m is not None for p in m.parameters()]
    opt = torch.optim.RMSprop(params, lr=0.00048, eps=0.01, alpha=0.99)
    b = batch_for(B, gaussian=False)
    state = tuple(torch.zeros(2, B, core, device="cuda") for _ in range(2))

    def step():
        x = torso(b["frame"])
        x = torch.cat([x, b["reward"].clamp(-1, 1)[..., None],
                       torch.nn.functional.one_hot(b["last_action"], 2 * D).float()], -1)
        if lstm is not None:
            notdone, s, ys = (~b["done"]).float(), state, []
            for t in range(T + 1):
                s = tuple(v * notdone[t][None, :, None] for v in s)
                y, s = lstm(x[t:t + 1], s)
                ys.append(y)
            x = torch.cat(ys, 0)
        logits, values = policy(x), baseline(x)[..., 0]
        disc = (~b["done"][1:]).float() * 0.99
        vs, pg_adv, _, _, _ = LT.vtrace_from_logits_torch(b["policy_logits"][1:], logits[:-1], b["action"][1:], disc,
                                                         b["reward"][1:].clamp(-1, 1), values[:-1], values[-1])
        total = sum(LT.impala_losses_torch(logits[:-1], b["action"][1:], pg_adv, vs, values[:-1], 0.5, 0.0006))
        opt.zero_grad()
        total.backward()
        torch.nn.utils.clip_grad_norm_(params, 40.0)
        opt.step()
        return total.item()
    return step


def kernel_graph(kind, obs, B=256):
    N = (T + 1) * B
    frame = torch.randn(T + 1, B, obs, device="cuda")
    mean = torch.zeros(obs, dtype=torch.float64, device="cuda")
    var, count = torch.ones_like(mean), torch.zeros_like(mean)
    ld = (obs + 7) // 8 * 8
    out = torch.empty(2 * N * ld, dtype=torch.bfloat16, device="cuda")
    sums = torch.zeros(3, obs, dtype=torch.float64, device="cuda")
    p, lib, st = _lib.ptr, _lib.lib(), _lib.stream_ptr

    def call():
        if kind == "stage":
            _lib.check(lib.tb_obs_stage(p(frame), N, obs, p(mean), p(var), 2, p(out), st()), "tb_obs_stage")
        elif kind == "sums":
            _lib.check(lib.tb_obs_norm_sums(p(frame), T + 1, B, obs, 1, B, p(sums), st()), "tb_obs_norm_sums")
        else:
            _lib.check(lib.tb_obs_norm_update(p(sums), p(count), p(mean), p(var), obs, st()), "tb_obs_norm_update")
    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            call()
    nbytes = {"stage": 4 * N * obs + 4 * N * ld + 16 * obs, "sums": 4 * T * B * obs + 24 * obs,
              "update": 72 * obs}[kind]
    return g, nbytes, (frame, mean, var, count, out, sums)


def acting_call(B):
    model = nets.MLPNet(O, Gaussian(D), hidden=HIDDEN, use_lstm=True, normalize_observations=True)
    model.train()
    model.action_sampler = ActionSampler(7)
    actor = GraphedActor(model)
    g = torch.Generator().manual_seed(B)
    inputs = dict(frame=torch.randn(1, B, O, generator=g).cuda(), reward=torch.zeros(1, B).cuda(),
                  done=torch.zeros(1, B, dtype=torch.bool).cuda(), last_action=torch.zeros(1, B, D).cuda())
    state = model.initial_state(B)

    def call():
        with torch.no_grad():
            return actor(inputs, state)
    return call


def report(res, unit="ms"):
    for name, xs in res.items():
        print("  %-34s median %8.3f %s  rounds %s" % (name, statistics.median(xs), unit,
                                                     ", ".join("%.3f" % x for x in xs)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mlpnet needs a GPU")
    print("card: %s" % card())
    print("\n1. graphed learn step, O=%d, Gaussian(%d), hidden %r, T=%d, ms per step" % (O, D, HIDDEN, T))
    for B in (32, 256):
        legs = {}
        for use_lstm in (False, True):
            for norm in (False, True):
                legs["B=%d lstm=%d norm=%d" % (B, use_lstm, norm)] = learn_step(B, use_lstm, norm)
        report(time_legs(legs, args.rounds, args.steps))
    print("\n2. staging and statistics kernels alone, T+1=%d, B=256, graphs of %d launches, us per launch"
          % (T + 1, LAUNCHES))
    for obs in (17, 376):
        legs = {kind: kernel_graph(kind, obs) for kind in ("stage", "sums", "update")}
        us = {kind: [] for kind in legs}
        for _ in range(args.rounds):
            for kind, (g, _b, _k) in legs.items():
                us[kind].append(time_graph(g) / LAUNCHES * 1e3)
        for kind, xs in us.items():
            m, nb = statistics.median(xs), legs[kind][1]
            print("  O=%-4d %-7s median %8.2f us  %8.3f MB  %7.1f GB/s  %5.1f%% of peak  rounds %s" % (
                obs, kind, m, nb * 1e-6, nb / m * 1e-3, 100 * nb / (m * 1e-6) / PEAK, ", ".join("%.2f" % x for x in xs)))
    print("\n3. graphed acting call, T=1, LSTM, normalisation on, ms per call")
    report(time_legs({"B=%d" % B: acting_call(B) for B in (1, 48, 512)}, args.rounds, args.steps * 4))
    print("\n4. plain torch (fp32 autograd, the oracle's V-trace, flat A=%d), ms per step" % (2 * D))
    legs = {"torch B=%d lstm=%d" % (B, use_lstm): torch_step(B, use_lstm) for B in (32, 256) for use_lstm in (False, True)}
    report(time_legs(legs, args.rounds, max(3, args.steps // 6)))


if __name__ == "__main__":
    main()
