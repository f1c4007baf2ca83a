"""Time the graphed learn step of the IMPALA ResNet (polybeast_learner.Net + LSTM, default bf16x3 backend,
learner.learn with flags.cuda_graph, T=80) with the paper's section widths (16, 32, 32) against "IMPALA x2"
(32, 64, 64), at the Atari stack (4, 84, 84) and Procgen (3, 64, 64), B = 8 and 32, in alternating rounds.  Prints
the card and its power limit, then ms/step and learner frames/s (T x B environment frames per step) per leg.

Then, for x2 at (4, 84, 84), B = 32: the device time of each 64-channel convolution (tb_profile_* records, one
learn step) with its algorithmic flops (2 x pixels x 9 x C_in x C_out; the split-bf16 product issues three times as
many on the tensor cores) and the bytes it must move, and which of the two H100 SXM data-sheet bounds applies
(989 TFLOP/s dense BF16, 3.35 TB/s HBM3).  Last, the same learn step in plain torch on cuDNN (oracle/learner_torch.
learner_step on CUDA tensors, fp32, TF32 off and on) for context.

    python tools/bench_resnet_width.py [--rounds 3] [--steps 20]
"""
import argparse
import collections
import os
import subprocess
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import _lib, learner, nets, optim, polybeast_learner  # noqa: E402

T, A = 80, 6
WIDTHS = [(16, 32, 32), (32, 64, 64)]
SHAPES = [(4, 84, 84), (3, 64, 64)]
PEAK_BF16, PEAK_HBM = 989e12, 3.35e12
FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def batch_for(obs, B, seed=2):
    batch = LT.synthetic_batch(T, B, A, seed=seed, with_last_action=False)
    batch["frame"] = torch.from_numpy(np.random.RandomState(seed + 1).randint(0, 256, size=(T + 1, B) + obs).astype(np.uint8))
    return batch


def leg(obs, channels, B):
    model = polybeast_learner.Net(A, True, observation_shape=obs, channels=channels)
    actor = polybeast_learner.Net(A, True, observation_shape=obs, channels=channels)
    model.reset_parameters_like_torch(seed=1)
    opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
    flags = types.SimpleNamespace(cuda_graph=True, **FLAGS)
    eager = types.SimpleNamespace(cuda_graph=False, **FLAGS)   # the per-op records are taken outside the graph
    batch = {k: v.cuda() for k, v in batch_for(obs, B).items()}
    state = model.initial_state(B)
    return (lambda: learner.learn(flags, model, actor, batch, state, opt, None),
            lambda: learner.learn(eager, model, actor, batch, state, opt, None))


def conv_table(obs, channels, N):
    """The convolutions of one learn step in the order the library records them: {(tag, k): (name, pixels, cin, cout,
    H, W)}.  Forward: per section the feat conv, then its four residual convs; backward: sections 2, 1, 0, each its four
    residual convs (weight gradient, then input gradient), then its feat conv."""
    C, H, W = obs
    hs, ws = [H], [W]
    for _ in range(3):
        hs.append((hs[-1] + 1) // 2)
        ws.append((ws[-1] + 1) // 2)
    cin = [16, channels[0], channels[1]]
    table, count = {}, collections.Counter()

    def add(tag, name, i, feat, c_in, c_out):
        h, w = (hs[i], ws[i]) if feat else (hs[i + 1], ws[i + 1])
        table[(tag, count[tag])] = (name, N * h * w, c_in, c_out, h, w)
        count[tag] += 1

    for i in range(3):
        add("feat_conv_fwd", "feat%d fwd" % i, i, True, cin[i], channels[i])
        for j in range(4):
            add("res_conv_fwd", "res%d.%d fwd" % (i, j), i, False, channels[i], channels[i])
    for i in (2, 1, 0):
        for j in (3, 2, 1, 0):
            add("res_conv_wgrad", "res%d.%d wgrad" % (i, j), i, False, channels[i], channels[i])
            add("res_conv_dgrad", "res%d.%d dgrad" % (i, j), i, False, channels[i], channels[i])
        if i > 0:
            add("res_conv_wgrad", "feat%d wgrad" % i, i, True, cin[i], channels[i])
            add("res_conv_dgrad", "feat%d dgrad" % i, i, True, channels[i], cin[i])
        else:
            add("feat_conv_wgrad", "feat0 wgrad", 0, True, cin[0], channels[0])
    return table


def conv_report(step, obs, channels, B):
    lib = _lib.lib()
    step()
    torch.cuda.synchronize()
    lib.tb_profile_enable(1)
    step()
    torch.cuda.synchronize()
    recs = _lib.profile_collect()
    lib.tb_profile_enable(0)
    table = conv_table(obs, channels, (T + 1) * B)
    count = collections.Counter()
    print("per-conv device time, %r at %dx%dx%d, B=%d (one eager learn step, tb_profile records):" % ((channels,) + obs + (B,)))
    print("  %-14s %-9s %9s %10s %9s %9s  %s" % ("conv", "C->O", "ms", "alg TFLOP", "TFLOP/s", "GB/s", "bound (share of it)"))
    for name, ms in recs:
        if "conv" not in name:
            continue
        key = (name, count[name])
        count[name] += 1
        if key not in table:
            continue
        label, pix, ci, co, h, w = table[key]
        if max(ci, co) < 64:
            continue
        flops = 2.0 * pix * 9 * ci * co
        padded = pix / (h * w) * (h + 2) * (w + 2)
        if "wgrad" in name:   # the dY and input images (hi + lo bf16)
            nbytes = 4.0 * padded * (ci + co)
        else:                 # the input image, the fp32 output (and at most one fp32 mask or residual read)
            nbytes = 4.0 * padded * ci + 8.0 * pix * co
        t = ms * 1e-3
        tf, tb = 3 * flops / PEAK_BF16, nbytes / PEAK_HBM
        bound = "tensor (%.0f %%)" % (100 * tf / t) if tf >= tb else "HBM (%.0f %%)" % (100 * tb / t)
        print("  %-14s %3d->%-3d %9.4f %10.4f %9.1f %9.0f  %s" % (label, ci, co, ms, flops / 1e12, flops / t / 1e12,
                                                                   nbytes / t / 1e9, bound))


def cudnn_step_ms(obs, channels, B, tf32, steps):
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    shapes = dict(nets.resnet_param_spec(A, True, observation_shape=obs, channels=channels))
    params = {k: v.cuda() for k, v in LT.random_params(shapes, seed=1).items()}
    batch = {k: v.cuda() for k, v in batch_for(obs, B).items()}
    state = tuple(torch.zeros(1, B, 256, device="cuda") for _ in range(2))
    hyper = type("H", (LT.Hyper,), dict(reward_clipping="abs_one"))
    for _ in range(2):
        LT.learner_step(params, batch, state, hyper=hyper, net="resnet", num_actions=A)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        LT.learner_step(params, batch, state, hyper=hyper, net="resnet", num_actions=A)
    torch.cuda.synchronize()
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch-sizes", default="8,32")
    ap.add_argument("--no-cudnn", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resnet_width needs a GPU")
    sizes = [int(b) for b in args.batch_sizes.split(",")]
    print("card: %s" % card(), flush=True)
    # the two widths of one (shape, B) alternate; only that pair is resident (x2 at B = 32 keeps a 28 GB workspace)
    for B in sizes:
        for obs in SHAPES:
            legs = {ch: leg(obs, ch, B) for ch in WIDTHS}
            for step, _ in legs.values():
                for _ in range(5):   # the graph capture and its warm-up
                    step()
            for r in range(args.rounds):
                for ch, (step, _) in legs.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(args.steps):
                        step()  # reads its stats back: one host sync per step, as in training
                    torch.cuda.synchronize()
                    ms = (time.perf_counter() - t0) * 1e3 / args.steps
                    print("round %d  obs %-9s channels %-13s B=%-3d %8.3f ms/step %10.0f frames/s"
                          % (r, "%dx%dx%d" % obs, "%d/%d/%d" % ch, B, ms, T * B / ms * 1e3), flush=True)
            if obs == (4, 84, 84) and B == max(sizes):
                conv_report(legs[WIDTHS[1]][1], obs, WIDTHS[1], B)
            del legs
            torch.cuda.empty_cache()
    if not args.no_cudnn:
        for (o, c, b) in [(o, c, b) for b in sizes for o in SHAPES for c in WIDTHS]:
            for tf32 in (False, True):
                ms = cudnn_step_ms(o, c, b, tf32, max(3, args.steps // 4))
                print("cuDNN (torch fp32, TF32 %s) obs %-9s channels %-13s B=%-3d %8.3f ms/step %10.0f frames/s"
                      % ("on " if tf32 else "off", "%dx%dx%d" % o, "%d/%d/%d" % c, b, ms, T * b / ms * 1e3), flush=True)
    print("card: %s" % card())


if __name__ == "__main__":
    main()
