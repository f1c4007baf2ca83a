"""Implicit-GEMM convolutions (wgmma + TMA gather) against torch.nn.functional.conv2d / torch.nn.grad in fp64
on the SAME bf16-rounded operands: the only differences left are fp32 accumulation order and the bf16 rounding
of the output, so the tolerances are tight (2^-8 relative for bf16 outputs, 1e-4*sqrt(K) for fp32 sums).
Shapes are AtariNet's conv2 / conv3 / conv1 (monobeast.py:560-562) with several frame counts (tile tails)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CONVS = [  # H, W, C, K, S, O
    (20, 20, 32, 4, 2, 64),   # conv2
    (9, 9, 64, 3, 1, 64),     # conv3
]
FRAMES = [1, 3, 50, 131]


def _bf16(x):
    return x.to(torch.bfloat16)


def _ptrs():
    from torchbeast_b200 import _lib
    return _lib, _lib.ptr, _lib.stream_ptr()


@pytest.mark.parametrize("H,W,C,K,S,O", CONVS)
@pytest.mark.parametrize("N", FRAMES)
def test_conv_forward(H, W, C, K, S, O, N):
    _lib, p, st = _ptrs()
    g = torch.Generator(device="cuda").manual_seed(N + H)
    x = _bf16(torch.randn(N, H, W, C, device="cuda", generator=g))          # NHWC
    w = torch.randn(O, C, K, K, device="cuda", generator=g) * 0.1
    b = torch.randn(O, device="cuda", generator=g)
    OH = (H - K) // S + 1
    out = torch.full((N, OH, OH, O), float("nan"), device="cuda").to(torch.bfloat16)
    pack = torch.empty(4 * O * C * K * K, device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib().tb_conv_nhwc_bf16_fwd(p(x), p(w), p(b), N, H, W, C, K, K, S, O, 1, p(out), p(pack), st), "fwd")
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), _bf16(w).double(), b.double(), stride=S).relu()
    ref = ref.permute(0, 2, 3, 1)
    torch.testing.assert_close(out.double(), ref, rtol=2 ** -7, atol=1e-3)


@pytest.mark.parametrize("H,W,C,K,S,O", CONVS)
@pytest.mark.parametrize("N", FRAMES)
def test_conv_input_gradient(H, W, C, K, S, O, N):
    _lib, p, st = _ptrs()
    g = torch.Generator(device="cuda").manual_seed(7 * N + H)
    OH = (H - K) // S + 1
    act = _bf16(torch.randn(N, H, W, C, device="cuda", generator=g))        # forward activation: ReLU mask = act > 0
    dy = _bf16(torch.randn(N, OH, OH, O, device="cuda", generator=g))
    w = torch.randn(O, C, K, K, device="cuda", generator=g) * 0.1
    dx = torch.full((N, H, W, C), float("nan"), device="cuda").to(torch.bfloat16)
    pack = torch.empty(4 * O * C * K * K, device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib().tb_conv_nhwc_bf16_dgrad(p(dy), p(w), p(act), N, H, W, C, K, K, S, O, p(dx), p(pack), st), "dgrad")
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_input((N, C, H, W), _bf16(w).double(), dy.double().permute(0, 3, 1, 2), stride=S)
    ref = ref.permute(0, 2, 3, 1) * (act.double() > 0)
    torch.testing.assert_close(dx.double(), ref, rtol=2 ** -7, atol=1e-3 * np.sqrt(K * K * O))


@pytest.mark.parametrize("H,W,C,K,S,O", CONVS)
@pytest.mark.parametrize("N", FRAMES)
def test_conv_weight_gradient(H, W, C, K, S, O, N):
    _lib, p, st = _ptrs()
    g = torch.Generator(device="cuda").manual_seed(13 * N + H)
    OH = (H - K) // S + 1
    act = _bf16(torch.randn(N, H, W, C, device="cuda", generator=g))
    dy = _bf16(torch.randn(N, OH, OH, O, device="cuda", generator=g))
    dw = torch.full((O, C, K, K), float("nan"), device="cuda")
    part = torch.empty(132 * O * C * K * K, device="cuda")  # one split per SM
    _lib.check(_lib.lib().tb_conv_nhwc_bf16_wgrad(p(dy), p(act), N, H, W, C, K, K, S, O, p(dw), p(part), part.numel(), st), "wgrad")
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_weight(act.double().permute(0, 3, 1, 2), (O, C, K, K), dy.double().permute(0, 3, 1, 2), stride=S)
    torch.testing.assert_close(dw.double(), ref, rtol=1e-4, atol=1e-4 * np.sqrt(N * OH * OH))


@pytest.mark.parametrize("N", [1, 5, 64])
def test_conv1_from_uint8_frames(N):
    """conv1 forward + weight gradient from uint8 NCHW frames (x/255 like the reference, monobeast.py:586-587)."""
    _lib, p, st = _ptrs()
    g = torch.Generator(device="cuda").manual_seed(N)
    frame = torch.randint(0, 256, (N, 4, 84, 84), device="cuda", generator=g, dtype=torch.uint8)
    w = torch.randn(32, 4, 8, 8, device="cuda", generator=g) * 0.05
    b = torch.randn(32, device="cuda", generator=g)
    out = torch.full((N, 20, 20, 32), float("nan"), device="cuda").to(torch.bfloat16)
    image = torch.empty(N * 4 * 84 * 84, device="cuda", dtype=torch.bfloat16)
    pack = torch.empty(32 * 256, device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib().tb_conv1_u8_fwd(p(frame), p(w), p(b), N, 84, 84, 4, 1, p(out), p(image), p(pack), st), "conv1 fwd")
    x = frame.double() / 255.0
    ref = torch.nn.functional.conv2d(x, _bf16(w).double(), b.double(), stride=4).relu().permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    torch.testing.assert_close(out.double(), ref, rtol=2 ** -7, atol=1e-3)
    dy = _bf16(torch.randn(N, 20, 20, 32, device="cuda", generator=g))
    dw = torch.full((32, 4, 8, 8), float("nan"), device="cuda")
    part = torch.empty(132 * 32 * 256, device="cuda")
    _lib.check(_lib.lib().tb_conv1_u8_wgrad(p(dy), p(image), N, 84, 84, 4, p(dw), p(part), part.numel(), st), "conv1 wgrad")
    torch.cuda.synchronize()
    refw = torch.nn.grad.conv2d_weight(x, (32, 4, 8, 8), dy.double().permute(0, 3, 1, 2), stride=4)
    torch.testing.assert_close(dw.double(), refw, rtol=1e-4, atol=1e-4 * np.sqrt(N * 400))
