"""The AtariNet trunk's tensor-core kernels in isolation at frame counts that leave partial tiles, against fp64 torch on
the same bf16 operands (tolerances as in test_conv_implicit_gpu.py).  conv_tc_kernel packs whole frames into its M tiles
and its two consumer warpgroups take alternate tiles: at 2592 frames (the learner's T=80, B=32 batch) 256-row tiles of 3
(conv2 forward, conv3 input gradient) or 5 (conv3 forward) frames, 128-row tiles of 1 or 2 frames at the small counts, and
one 100-pixel frame per tile for conv2's stride-2 input gradient.  The weight gradient packs whole frames into its pipeline
stages.  Frame counts from one frame up are checked, each with a last tile or stage holding fewer frames than the others and
with an odd or even number of tiles per CTA.  The input-gradient cases run the ReLU-mask epilogue; the dense cases run
gemm_tc_kernel's bias / ReLU epilogue with fp32 and bf16 outputs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CONVS = [  # H, W, C, K, S, O
    (20, 20, 32, 4, 2, 64),   # conv2: 81 patches per frame, input gradient in 4 parity classes of 100 pixels
    (9, 9, 64, 3, 1, 64),     # conv3: 49 patches per frame, input gradient over 81 pixels
]
FRAMES = [1, 2, 4, 7, 2591, 2592]  # 2591: a last 256-row tile of 2 frames (conv2 forward, conv3 input gradient)


def _bf16(x):
    return x.to(torch.bfloat16)


def _lib_ptrs():
    from torchbeast_b200 import _lib
    return _lib, _lib.ptr, _lib.stream_ptr()


@pytest.mark.parametrize("H,W,C,K,S,O", CONVS)
@pytest.mark.parametrize("N", FRAMES)
def test_forward_tail_tiles(H, W, C, K, S, O, N):
    _lib, p, st = _lib_ptrs()
    g = torch.Generator(device="cuda").manual_seed(3 * N + H)
    x = _bf16(torch.randn(N, H, W, C, device="cuda", generator=g))
    w = torch.randn(O, C, K, K, device="cuda", generator=g) * 0.1
    b = torch.randn(O, device="cuda", generator=g)
    OH = (H - K) // S + 1
    out = torch.full((N, OH, OH, O), float("nan"), device="cuda").to(torch.bfloat16)
    pack = torch.empty(4 * O * C * K * K, device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib().tb_conv_nhwc_bf16_fwd(p(x), p(w), p(b), N, H, W, C, K, K, S, O, 1, p(out), p(pack), st), "fwd")
    torch.cuda.synchronize()
    ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), _bf16(w).double(), b.double(), stride=S).relu()
    torch.testing.assert_close(out.double(), ref.permute(0, 2, 3, 1), rtol=2 ** -7, atol=1e-3)


@pytest.mark.parametrize("H,W,C,K,S,O", CONVS)
@pytest.mark.parametrize("N", FRAMES)
def test_input_gradient_tail_tiles(H, W, C, K, S, O, N):
    _lib, p, st = _lib_ptrs()
    g = torch.Generator(device="cuda").manual_seed(5 * N + H)
    OH = (H - K) // S + 1
    act = _bf16(torch.randn(N, H, W, C, device="cuda", generator=g))  # ReLU mask = act > 0
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
def test_weight_gradient_tail_stages(H, W, C, K, S, O, N):
    _lib, p, st = _lib_ptrs()
    g = torch.Generator(device="cuda").manual_seed(11 * N + H)
    OH = (H - K) // S + 1
    act = _bf16(torch.randn(N, H, W, C, device="cuda", generator=g))
    dy = _bf16(torch.randn(N, OH, OH, O, device="cuda", generator=g))
    dw = torch.full((O, C, K, K), float("nan"), device="cuda")
    part = torch.empty(132 * O * C * K * K, device="cuda")
    _lib.check(_lib.lib().tb_conv_nhwc_bf16_wgrad(p(dy), p(act), N, H, W, C, K, K, S, O, p(dw), p(part), part.numel(), st), "wgrad")
    torch.cuda.synchronize()
    ref = torch.nn.grad.conv2d_weight(act.double().permute(0, 3, 1, 2), (O, C, K, K), dy.double().permute(0, 3, 1, 2), stride=S)
    torch.testing.assert_close(dw.double(), ref, rtol=1e-4, atol=1e-4 * np.sqrt(N * OH * OH))


# M = 1 and 2: the acting forward's single partial tile; 3 * 128 + 1: a one-row last tile
@pytest.mark.parametrize("M", [1, 2, 385, 2592])
@pytest.mark.parametrize("N,K", [(512, 3136), (64, 576), (2076, 520)])
def test_dense_tail_tiles(M, N, K):
    from torchbeast_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    B = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=g)
    C = torch.full((M, N), float("nan"), device="cuda")
    C16 = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    p = _lib.ptr
    _lib.check(_lib.lib().tb_gemm_bf16_tn(p(A), p(B), M, N, K, K, K, p(C), N, p(C16), N, p(bias), 1.0, 1, _lib.stream_ptr()),
               "tb_gemm_bf16_tn")
    torch.cuda.synchronize()
    ref = (A.double() @ B.double().t() + bias.double()).clamp(min=0)
    torch.testing.assert_close(C.double(), ref, rtol=1e-4, atol=1e-4 * np.sqrt(K))
    torch.testing.assert_close(C16.double(), ref, rtol=2 ** -7, atol=1e-3)
