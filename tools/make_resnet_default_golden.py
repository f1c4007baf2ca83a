"""Write tests/golden/resnet_obs_default_bits.npz: the exact float32 results of the ResNet's (4, 84, 84) path with the
default widths through tb_resnet_forward / tb_resnet_backward on each backend, ±LSTM, at T1=3, B=2 (policy logits, baseline,
hN and 4096 strided samples of the parameter gradients).  The committed file was written by the build that had no
observation geometry (fixed 84 x 84 constants); tests/test_resnet_obs_gpu.py checks that the current build reproduces it
bit for bit on an H100.

    python tools/make_resnet_default_golden.py [OUT]
"""
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import learner_torch as LT  # noqa: E402
from torchbeast_b200 import _lib  # noqa: E402

A, T1, B, SAMPLES = 6, 3, 2, 4096


def default_case(use_lstm, precision):
    """(logits, baseline, hN or empty, strided gradient samples) of the fixed (4, 84, 84) case."""
    lib = _lib.lib()
    p = lambda t: None if t is None else ctypes.c_void_p(t.data_ptr())
    params = torch.cat([v.flatten() for v in LT.random_params(LT.resnet_param_shapes(A, use_lstm), seed=2).values()]).cuda()
    rs = np.random.RandomState(4)
    frame = torch.from_numpy(rs.randint(0, 256, size=(T1, B, 4, 84, 84)).astype(np.uint8)).cuda()
    reward = torch.from_numpy(rs.randn(T1, B).astype(np.float32)).cuda()
    notdone = torch.from_numpy((rs.rand(T1, B) > 0.3).astype(np.float32)).cuda() if use_lstm else None
    h0 = torch.from_numpy(rs.randn(1, B, 256).astype(np.float32) * 0.1).cuda() if use_lstm else None
    c0 = torch.from_numpy(rs.randn(1, B, 256).astype(np.float32) * 0.1).cuda() if use_lstm else None
    hN = torch.empty(1, B, 256, device="cuda") if use_lstm else None
    cN = torch.empty(1, B, 256, device="cuda") if use_lstm else None
    logits = torch.empty(T1, B, A, device="cuda")
    baseline = torch.empty(T1, B, device="cuda")
    gl = torch.from_numpy(rs.randn(T1, B, A).astype(np.float32)).cuda()
    gb = torch.from_numpy(rs.randn(T1, B).astype(np.float32)).cuda()
    grads = torch.empty_like(params)
    geometry = (4, 84, 84, 16, 32, 32)
    ws = torch.empty(lib.tb_resnet_workspace_bytes(*geometry, T1, B, A, int(use_lstm), precision), dtype=torch.uint8,
                     device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.tb_resnet_forward(p(frame), None, p(reward), p(notdone), p(h0), p(c0), p(params), *geometry, T1, B, A, 1,
                                     int(use_lstm), precision, p(ws), None, p(logits), p(baseline), p(hN), p(cN), st),
               "tb_resnet_forward")
    _lib.check(lib.tb_resnet_backward(p(frame), p(gl), p(gb), p(notdone), p(params), *geometry, T1, B, A, 1, int(use_lstm),
                                      precision, p(ws), p(grads), st), "tb_resnet_backward")
    idx = torch.linspace(0, params.numel() - 1, SAMPLES).long().cuda()
    return {"logits": logits.cpu().numpy(), "baseline": baseline.cpu().numpy(),
            "hN": hN.cpu().numpy() if use_lstm else np.zeros(0, np.float32), "grads": grads[idx].cpu().numpy()}


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "resnet_obs_default_bits.npz")
    arrays = {}
    for use_lstm in (False, True):
        for precision in (0, 1, 2):
            for k, v in default_case(use_lstm, precision).items():
                arrays["%s/lstm%d/p%d" % (k, use_lstm, precision)] = v
    np.savez_compressed(out, **arrays)
    print("wrote", out)


if __name__ == "__main__":
    main()
