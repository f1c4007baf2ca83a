"""Acting-forward timing: the training-mode forward an inference thread runs per environment step (T=1) at B in
{1, 48, 512} actors, once with the seeded sampler attached (torchbeast_b200.sampling.ActionSampler), once with the
reference's torch.multinomial(softmax(.)) and once replayed as a CUDA graph with the sampler attached
(torchbeast_b200.acting.GraphedActor), plus each sampling step on its own.

    python tools/bench_acting.py [--net atari|resnet] [--use_lstm 0|1] [--precision fp32|bf16|bf16x3] [--num_actions A]

Calls back to back (host launch cost included, as an inference thread pays it), CUDA events around `--reps` calls;
the five measurements alternate over `--rounds` rounds and each number is the median round.  Prints one JSON line with an
`acting` key, beside the card's name and power limit (an absolute time means nothing without them).  Writes no files.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card_info(index):
    info = dict(name=torch.cuda.get_device_name(index), power_limit_w=None)
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return info


def acting_batch(B, A, seed):
    """One synthetic [1, B, ...] acting step (numpy RandomState), on the GPU."""
    rs = np.random.RandomState(seed)
    return dict(
        frame=torch.from_numpy(rs.randint(0, 256, size=(1, B, 4, 84, 84), dtype=np.uint8)).cuda(),
        reward=torch.from_numpy(rs.randn(1, B).astype(np.float32)).cuda(),
        done=torch.from_numpy(rs.rand(1, B) < 0.01).cuda(),
        last_action=torch.from_numpy(rs.randint(0, A, size=(1, B)).astype(np.int64)).cuda(),
    )


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", default="atari", choices=["atari", "resnet"])
    ap.add_argument("--use_lstm", type=int, default=1)
    ap.add_argument("--precision", default=None, choices=["fp32", "bf16", "bf16x3"])
    ap.add_argument("--num_actions", type=int, default=6)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_acting.py needs a GPU (there is no CPU fallback)"
    torch.cuda.set_device(0)
    from torchbeast_b200 import monobeast, polybeast_learner
    from torchbeast_b200.acting import GraphedActor
    from torchbeast_b200.sampling import ActionSampler

    A, use_lstm = args.num_actions, bool(args.use_lstm)
    if args.net == "resnet":
        model = polybeast_learner.Net(A, use_lstm, precision=args.precision)
    else:
        model = monobeast.AtariNet((4, 84, 84), A, use_lstm, precision=args.precision)
    model.reset_parameters_like_torch(seed=0)
    model.train()
    sampler = ActionSampler(seed=0)

    def per_call_ms(fn):
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            fn()
        z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z) / args.reps

    def forward_with(s, batch, state):
        def run():
            model.action_sampler = s
            return model(batch, state)
        return run

    graphed = GraphedActor(model)

    def graphed_with(s, batch, state):
        def run():
            model.action_sampler = s
            return graphed(batch, state)
        return run

    cases = []
    with torch.no_grad():
        for B in (1, 48, 512):
            batch = acting_batch(B, A, seed=B)
            state = model.initial_state(B)
            logits = model.learner_forward(batch, state).policy_logits
            fns = dict(
                acting_sampler=forward_with(sampler, batch, state), acting_torch=forward_with(None, batch, state),
                acting_graphed=graphed_with(sampler, batch, state),
                sample_sampler=lambda: sampler.sample(logits),
                sample_torch=lambda: torch.multinomial(torch.softmax(logits.view(B, A), dim=1), num_samples=1))
            for fn in fns.values():  # warm-up: module loads, allocator, library heuristics
                for _ in range(5):
                    fn()
            times = {k: [] for k in fns}
            for _ in range(args.rounds):
                for k, fn in fns.items():
                    times[k].append(per_call_ms(fn))
            med = {k: float(np.median(v)) for k, v in times.items()}
            cases.append(dict(B=B, acting_ms_sampler=med["acting_sampler"], acting_ms_torch=med["acting_torch"],
                              acting_ms_graphed=med["acting_graphed"], sample_us_sampler=med["sample_sampler"] * 1e3, sample_us_torch=med["sample_torch"] * 1e3,
                              logits_bytes=4 * B * A, actions_bytes=8 * B))
    model.action_sampler = None
    print(json.dumps(dict(acting=dict(
        net=args.net, use_lstm=use_lstm, precision=model.precision, T=1, num_actions=A, card=card_info(0),
        timing="%d eager calls per CUDA-event pair, median of %d alternating rounds" % (args.reps, args.rounds),
        cases=cases))))


if __name__ == "__main__":
    main()
