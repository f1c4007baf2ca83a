"""Cost of the state-gradient ports of the standalone LSTM backward, measured in alternating rounds.

    python tools/bench_lstm_state.py [--rounds 3] [--steps 20]

For each shape it times tb_lstm_backward against tb_lstm_backward_state with all four ports set (dhN, dcN in; dh0, dc0
out) after one tb_lstm_forward on the same workspace, CUDA events around `--steps` calls after a warm-up:
  * AtariNet's core: T1 = 81, B = 32, 2 layers of 519, bf16x3 (the wavefront kernels);
  * ResNet's core: T1 = 81, B = 8, 257 -> 256, bf16x3 (the cluster kernels);
  * BASELINE configs[4]: T1 = 601, B = 128, 512 -> 512, fp32 (the step kernels).
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
    ("atarinet_core", 81, 32, 519, 519, 2, "bf16x3"),
    ("resnet_core", 81, 8, 257, 256, 1, "bf16x3"),
    ("configs[4]", 601, 128, 512, 512, 1, "fp32"),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit unknown"
    return "%s (%s)" % (torch.cuda.get_device_name(0), q)


def timed(fn, steps, warmup=3):
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
    """Runs one forward; returns (backward without ports, backward with all four ports) as closures, and the plan."""
    lib, p = _lib.lib(), _lib.ptr
    prec = tl.PRECISIONS[precision]
    m = tl.LSTM(In, H, layers, precision=precision)
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    x, nd = rnd(T1, B, In) * 0.5, (torch.rand(T1, B, device="cuda", generator=g) > 0.02).float()
    h0, c0, dhN, dcN = (rnd(layers, B, H) * 0.1 for _ in range(4))
    dy = rnd(T1, B, H)
    arr = lambda ts: ctypes.cast(m._ptr_array(ts), ctypes.c_void_p)  # noqa: E731
    params = [q.detach().contiguous() for q in m._plist()]
    grads = [torch.empty_like(q) for q in params]
    ws = torch.empty(lib.tb_lstm_workspace_bytes(T1, B, In, H, layers, prec), dtype=torch.uint8, device="cuda")
    y, hN, cN = torch.empty(T1, B, H, device="cuda"), torch.empty(layers, B, H, device="cuda"), torch.empty_like(h0)
    dx, dh0, dc0 = torch.empty_like(x), torch.empty_like(h0), torch.empty_like(h0)
    _lib.check(lib.tb_lstm_forward(p(x), p(nd), p(h0), p(c0), arr(params), T1, B, In, H, layers, prec, p(ws), p(y), p(hN),
                                   p(cN), _lib.stream_ptr()), "tb_lstm_forward")
    pa, ga = arr(params), arr(grads)

    def base():
        _lib.check(lib.tb_lstm_backward(p(dy), p(x), p(nd), pa, ga, T1, B, In, H, layers, prec, p(ws), p(dx),
                                        _lib.stream_ptr()), "tb_lstm_backward")

    def ports():
        _lib.check(lib.tb_lstm_backward_state(p(dy), p(x), p(nd), pa, ga, T1, B, In, H, layers, prec, p(ws), p(dx), p(dhN),
                                              p(dcN), p(dh0), p(dc0), _lib.stream_ptr()), "tb_lstm_backward_state")
    return base, ports, m.plan(B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lstm_state measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    print("card: %s" % card(), flush=True)
    for name, T1, B, In, H, layers, precision in SHAPES:
        base, ports, plan = setup(T1, B, In, H, layers, precision)
        for r in range(args.rounds):
            order = (("base", base), ("ports", ports)) if r % 2 == 0 else (("ports", ports), ("base", base))
            ms = {k: timed(fn, args.steps) for k, fn in order}
            print(json.dumps(dict(round=r, shape=name, T1=T1, B=B, In=In, H=H, layers=layers, precision=precision,
                                  kinds=list(plan), backward_ms=round(ms["base"], 4), backward_state_ms=round(ms["ports"], 4),
                                  overhead_pct=round(100.0 * (ms["ports"] / ms["base"] - 1.0), 2))), flush=True)


if __name__ == "__main__":
    main()
