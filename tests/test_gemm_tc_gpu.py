"""GPU: the wgmma/TMA bf16 GEMM against a plain PyTorch fp32 reference of the same op
(inputs rounded to bf16 first, so products are exact and only the fp32 accumulation order differs:
tolerance rtol 1e-4 / atol 1e-4 x sqrt(K))."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [
    (128, 64, 64), (128, 32, 256), (256, 64, 512), (1000, 64, 576), (300, 32, 256), (129, 70, 200),
    (2592, 512, 3136), (64, 128, 64), (5, 6, 520), (4000, 2076, 520), (2592 * 4, 32, 256), (128, 200, 72),
]


def run(M, N, K, bias, relu, scale, want16):
    from torchbeast_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    B = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    bvec = torch.randn(N, device="cuda", generator=g) if bias else None
    C = torch.full((M, N), float("nan"), device="cuda")
    C16 = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16) if want16 else None
    p = _lib.ptr
    rc = _lib.lib().tb_gemm_bf16_tn(p(A), p(B), M, N, K, K, K, p(C), N, p(C16), N, p(bvec), scale, int(relu), _lib.stream_ptr())
    _lib.check(rc, "tb_gemm_bf16_tn")
    torch.cuda.synchronize()
    ref = (A.float() @ B.float().t()) * scale
    if bias:
        ref = ref + bvec
    if relu:
        ref = ref.clamp(min=0)
    return C, C16, ref


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_tc_matches_fp32_reference(M, N, K):
    if K % 8:
        pytest.skip("ld must be a multiple of 8")
    C, _, ref = run(M, N, K, bias=False, relu=False, scale=1.0, want16=False)
    tol = 1e-4 * np.sqrt(K)
    assert torch.isfinite(C).all()
    torch.testing.assert_close(C, ref, rtol=1e-4, atol=tol)


@pytest.mark.parametrize("M,N,K", [(300, 64, 512), (2592, 512, 3136), (1000, 32, 256)])
def test_gemm_tc_epilogue(M, N, K):
    C, C16, ref = run(M, N, K, bias=True, relu=True, scale=1.0 / 255.0, want16=True)
    torch.testing.assert_close(C, ref, rtol=1e-4, atol=1e-4 * np.sqrt(K))
    torch.testing.assert_close(C16.float(), ref, rtol=1e-2, atol=1e-2)


def test_f32_to_bf16_padding():
    from torchbeast_b200 import _lib
    x = torch.randn(37, 519, device="cuda")
    out = torch.full((37, 520), 7.0, device="cuda", dtype=torch.bfloat16)
    _lib.check(_lib.lib().tb_f32_to_bf16(_lib.ptr(x), _lib.ptr(out), 37, 519, 519, 520, _lib.stream_ptr()), "cvt")
    assert torch.equal(out[:, :519], x.to(torch.bfloat16)) and float(out[:, 519].abs().sum()) == 0.0


EX_SHAPES = [(128, 64, 64), (128, 128, 128), (256, 64, 512), (1000, 512, 64), (300, 576, 64), (64, 256, 4096),
             (32, 256, 20000), (512, 3136, 2592), (2076, 520, 2592), (6, 520, 2592), (129, 70 * 8, 200)]


@pytest.mark.parametrize("M,N,K", EX_SHAPES)
@pytest.mark.parametrize("mode", ["dgrad", "wgrad", "wgrad_splitk"])
def test_gemm_tc_mn_major_operands(M, N, K, mode):
    """dgrad form (A K-major, B stored [K,N]) and wgrad form (A stored [K,M], B stored [K,N])."""
    from torchbeast_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a_mn = mode != "dgrad"
    if (N % 8) or (a_mn and M % 8) or ((not a_mn) and K % 8):
        pytest.skip("leading dimensions must be multiples of 8")
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g).to(torch.bfloat16)
    B = torch.randn(K, N, device="cuda", generator=g).to(torch.bfloat16)
    C = torch.full((M, N), float("nan"), device="cuda")
    splits = 7 if mode == "wgrad_splitk" else 1
    part = torch.empty(splits * M * ((N + 31) // 32 * 32), device="cuda") if splits > 1 else None  # rows padded to 32 floats
    p = _lib.ptr
    rc = _lib.lib().tb_gemm_bf16_ex(p(A), p(B), M, N, K, A.shape[1], N, int(a_mn), 1, p(C), N, splits, p(part), _lib.stream_ptr())
    _lib.check(rc, "tb_gemm_bf16_ex")
    torch.cuda.synchronize()
    ref = (A.float().t() if a_mn else A.float()) @ B.float()
    torch.testing.assert_close(C, ref, rtol=1e-4, atol=1e-4 * np.sqrt(K))
