"""Per-op device time of the learner step, every op tag: a few eager steps under tb_profile_enable (CUDA events around
every op on its stream, as bench.py's roofline table), printed as ms per step sorted by time, with the card name and
power limit the numbers belong to.

    python tools/prof_ops.py [--T 80] [--B 32] [--steps 5] [--warmup 3] [--net atari|resnet] [--json FILE]

Ops that run on the side stream overlap the main stream, so the column does not add up to the step time."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import flags_ns, synthetic_host_batch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # the numbers still stand, without the card line
        out = "nvidia-smi unavailable (%s)" % exc
    return out or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=80)
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--num_actions", type=int, default=6)
    ap.add_argument("--net", default="atari", choices=["atari", "resnet"])
    ap.add_argument("--precision", default=None, choices=["fp32", "bf16", "bf16x3"])
    ap.add_argument("--steps", type=int, default=5, help="profiled steps")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the table to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "prof_ops.py needs a GPU"
    from torchbeast_b200 import _lib, learner, monobeast, optim, polybeast_learner

    T, B, A = args.T, args.B, args.num_actions
    if args.net == "resnet":
        model = polybeast_learner.Net(A, True, precision=args.precision)
        actor = polybeast_learner.Net(A, True, precision=args.precision)
    else:
        model = monobeast.AtariNet((4, 84, 84), A, True, precision=args.precision)
        actor = monobeast.AtariNet((4, 84, 84), A, True, precision=args.precision)
    model.reset_parameters_like_torch(seed=0)
    actor.copy_params_from(model)
    opt = optim.RMSprop(model, lr=0.00048, momentum=0, eps=0.01, alpha=0.99)
    flags = flags_ns(T, B)
    state = model.initial_state(B)
    batches = [{k: v.cuda() for k, v in synthetic_host_batch(T, B, A, seed=i, pin=False).items()} for i in range(2)]
    lib = _lib.lib()
    for i in range(args.warmup):
        learner.learn_step(flags, model, actor, batches[i % 2], state, opt, None, stats_sync=False)
    torch.cuda.synchronize()
    lib.tb_profile_enable(1)
    for i in range(args.steps):
        learner.learn_step(flags, model, actor, batches[i % 2], state, opt, None, stats_sync=False)
    recs = _lib.profile_collect()
    lib.tb_profile_enable(0)
    agg = {}
    for name, t in recs:
        a = agg.setdefault(name, [0.0, 0])
        a[0] += t
        a[1] += 1
    rows = sorted(((n, tot / args.steps, cnt / args.steps) for n, (tot, cnt) in agg.items()), key=lambda r: -r[1])
    info = dict(card=card(), net=args.net, precision=model.precision, T=T, B=B, steps=args.steps)
    print("# %s | %s %s T=%d B=%d, %d eager steps" % (info["card"], args.net, model.precision, T, B, args.steps))
    print("%-36s %10s %10s" % ("op", "ms/step", "launches"))
    for n, ms, cnt in rows:
        print("%-36s %10.4f %10.1f" % (n, ms, cnt))
    print("%-36s %10.4f" % ("(sum over ops)", sum(r[1] for r in rows)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(info, ops=[dict(op=n, ms_per_step=ms, launches_per_step=c) for n, ms, c in rows]), f, indent=1)


if __name__ == "__main__":
    main()
