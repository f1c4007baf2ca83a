"""Time the V-trace scan and the fused loss kernel over a size sweep (CUDA events on the
launch stream, L2 flushed between iterations) and report achieved algorithmic GB/s against
MEASURED_PEAKS.json.  Writes gpurun_out/vtrace_sweep.json.  (SURVEY.md 8(d) M4.)"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from torchbeast_b200 import _lib, learner  # noqa: E402
from torchbeast_b200.core import vtrace  # noqa: E402


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"], "measured"
    except Exception:
        return 3350.0, "H100 SXM data sheet"


def time_graphed(fn, reps=20, iters=10):
    """Device-side time per launch: `reps` launches captured in one CUDA graph, replayed `iters` times."""
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3): fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps): fn()
    ts = []
    for _ in range(iters):
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); g.replay(); z.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(z) * 1e3 / reps)
    return sorted(ts)[len(ts) // 2]


def time_kernel(fn, iters, flush=None):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    for s, e in ev:
        if flush is not None:
            flush.add_(1)
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    ts = sorted(s.elapsed_time(e) * 1e3 for s, e in ev)  # us
    return ts[len(ts) // 2], ts[0]


def main():
    torch.cuda.set_device(0)
    peak, how = peaks()
    flush = torch.zeros(256 * 1024 * 1024 // 4, device="cuda")  # 256 MB > 50 MB L2
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    A = 6
    sizes = [(80, 4), (80, 32), (80, 64), (600, 128)] + [(80, 1 << k) for k in range(10, 21, 2)] + [(80, 1 << 21)]
    for T, B in sizes:
        lr = 0.5 * torch.randn(T, B, device="cuda", generator=g)
        dc = 0.99 * (torch.rand(T, B, device="cuda", generator=g) > 0.01).float()
        rw = torch.randn(T, B, device="cuda", generator=g).clamp(-1, 1)
        va = torch.randn(T, B, device="cuda", generator=g)
        bs = torch.randn(B, device="cuda", generator=g)
        vs = torch.empty_like(va); pg = torch.empty_like(va)
        lib = _lib.lib()
        p = _lib.ptr

        def scan():
            lib.tb_vtrace_from_importance_weights_f32(p(lr), p(dc), p(rw), p(va), p(bs), T, B, 1.0, 1.0, p(vs), p(pg), _lib.stream_ptr())

        iters = 50 if T * B < (1 << 24) else 10
        med, best = time_kernel(scan, iters, flush)
        med_hot, best_hot = time_kernel(scan, iters, None)
        nbytes = 24 * T * B + 4 * B
        us_graph = time_graphed(scan) if T * B <= (1 << 22) else None  # device time per launch, inputs L2-hot
        row = dict(kernel="vtrace_scan", T=T, B=B, bytes=nbytes, us_median=med, us_best=best, us_hot_median=med_hot,
                   us_graphed_hot=us_graph, gbs=nbytes / med / 1e3, frac=nbytes / med / 1e3 / peak)
        rows.append(row); print(json.dumps(row), flush=True)
        if T * B * A * 4 * 3 > 8e9:
            continue
        bl = torch.randn(T, B, A, device="cuda", generator=g); tl = torch.randn(T, B, A, device="cuda", generator=g)
        ac = torch.randint(0, A, (T, B), device="cuda", generator=g)
        dn = torch.rand(T, B, device="cuda", generator=g) < 0.01
        outs = [torch.empty_like(va) for _ in range(5)]
        losses = torch.empty(4, device="cuda"); gl = torch.empty(T + 1, B, A, device="cuda"); gv = torch.empty(T + 1, B, device="cuda")
        ws = _lib.workspace(); dnu = dn.view(torch.uint8)

        def fused():
            lib.tb_impala_loss_f32(p(bl), p(tl), p(ac), p(rw), p(dnu), None, p(va), p(bs), T, B, A, 0.99, 0.5, 0.0006,
                                   1, 1.0, 1.0, *[None] * 5, 0, *[None] * 4, *[p(o) for o in outs], p(losses), p(gl), p(gv), 1,
                                   p(ws), _lib.stream_ptr())

        med, best = time_kernel(fused, iters, flush)
        med_hot, _ = time_kernel(fused, iters, None)
        nbytes = (12 * A + 32 + 12 - 3) * T * B + 4 * B + 16  # done is 1 byte (not 4): (12A+32)-3, +12 for log_rhos/alp outputs
        us_graph = time_graphed(fused) if T * B <= (1 << 22) else None
        row = dict(kernel="impala_loss_fwd_bwd", T=T, B=B, A=A, bytes=nbytes, us_median=med, us_best=best,
                   us_hot_median=med_hot, us_graphed_hot=us_graph, gbs=nbytes / med / 1e3, frac=nbytes / med / 1e3 / peak)
        rows.append(row); print(json.dumps(row), flush=True)
        del bl, tl, ac, dn, outs, gl, gv
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(dict(peak_gbs=peak, peak_source=how, rows=rows), open(os.path.join(ROOT, "gpurun_out", "vtrace_sweep.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
