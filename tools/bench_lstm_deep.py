"""Forward + backward time of stacks deeper than two layers, beside torch.nn.LSTM (cuDNN) of the same depth.

    python tools/bench_lstm_deep.py [--rounds 3] [--steps 10] [--warmup 3]

One call is tb_lstm_forward then tb_lstm_backward on the same workspace; the cuDNN call is torch.nn.LSTM's forward over
the whole sequence (no reset mask: cuDNN has none) and its backward to the input and every parameter, in fp32 with torch's
default cuDNN settings.  Each round times `--steps` calls of each, on CUDA events after a warm-up, in alternating order.
Shapes:
  * four layers of 519, T1 = 81, B = 32, bf16x3: two split-bf16 wavefront segments (AtariNet's core made deeper);
  * three layers, 257 -> 256, T1 = 81, B = 8, bf16x3 (ResNet's core made deeper);
  * three layers, 512 -> 512, T1 = 601, B = 128, fp32 (BASELINE configs[4] made deeper).
The card's name and power limit are printed first: the numbers belong to them.  Writes nothing.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchbeast_b200 import _lib  # noqa: E402
from torchbeast_b200 import lstm as tl  # noqa: E402

SHAPES = [  # name, T1, B, In, H, layers, precision
    ("atarinet_core_x4", 81, 32, 519, 519, 4, "bf16x3"),
    ("resnet_core_x3", 81, 8, 257, 256, 3, "bf16x3"),
    ("configs[4]_x3", 601, 128, 512, 512, 3, "fp32"),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (torch.cuda.get_device_name(0), q)


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def setup(T1, B, In, H, layers, precision):
    """Returns (this project's forward + backward, cuDNN's forward + backward) as closures, and the per-layer plan."""
    lib, p = _lib.lib(), _lib.ptr
    prec = tl.PRECISIONS[precision]
    m = tl.LSTM(In, H, layers, precision=precision)
    ref = torch.nn.LSTM(In, H, num_layers=layers).cuda()
    ref.load_state_dict(m.state_dict())
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    x, nd = rnd(T1, B, In) * 0.5, (torch.rand(T1, B, device="cuda", generator=g) > 0.02).float()
    h0, c0 = rnd(layers, B, H) * 0.1, rnd(layers, B, H) * 0.1
    dy = rnd(T1, B, H)
    arr = lambda ts: ctypes.cast(m._ptr_array(ts), ctypes.c_void_p)  # noqa: E731
    params = [q.detach().contiguous() for q in m._plist()]
    grads = [torch.empty_like(q) for q in params]
    ws = torch.empty(lib.tb_lstm_workspace_bytes(T1, B, In, H, layers, prec), dtype=torch.uint8, device="cuda")
    y, hN, cN = torch.empty(T1, B, H, device="cuda"), torch.empty_like(h0), torch.empty_like(h0)
    dx = torch.empty_like(x)
    pa, ga = arr(params), arr(grads)

    def ours():
        _lib.check(lib.tb_lstm_forward(p(x), p(nd), p(h0), p(c0), pa, T1, B, In, H, layers, prec, p(ws), p(y), p(hN),
                                       p(cN), _lib.stream_ptr()), "tb_lstm_forward")
        _lib.check(lib.tb_lstm_backward(p(dy), p(x), p(nd), pa, ga, T1, B, In, H, layers, prec, p(ws), p(dx),
                                        _lib.stream_ptr()), "tb_lstm_backward")

    xr = x.clone().requires_grad_(True)

    def cudnn():
        out, _ = ref(xr, (h0, c0))
        torch.autograd.backward(out, dy)
        xr.grad = None
        ref.zero_grad(set_to_none=True)
    return ours, cudnn, m.plan_layers(B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lstm_deep measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    print("card: %s; cudnn %s, cudnn.allow_tf32=%s" % (card(), torch.backends.cudnn.version(),
                                                       torch.backends.cudnn.allow_tf32), flush=True)
    for name, T1, B, In, H, layers, precision in SHAPES:
        ours, cudnn, plan = setup(T1, B, In, H, layers, precision)
        for r in range(args.rounds):
            order = (("ours", ours), ("cudnn", cudnn)) if r % 2 == 0 else (("cudnn", cudnn), ("ours", ours))
            ms = {k: timed(fn, args.steps, args.warmup) for k, fn in order}
            print(json.dumps(dict(round=r, shape=name, T1=T1, B=B, In=In, H=H, layers=layers, precision=precision,
                                  kinds=[list(k) for k in plan], fwd_bwd_ms=round(ms["ours"], 3),
                                  cudnn_fp32_fwd_bwd_ms=round(ms["cudnn"], 3))), flush=True)


if __name__ == "__main__":
    main()
