"""CPU: the reference helpers of tests/sw_image.py against torch's own operators, so that a failure of the GPU convolution
tests points at a kernel and not at its reference."""
import pytest
import torch

from tests import sw_image as S


def test_split_is_rne_hi_and_rne_residual():
    x = torch.randn(4096, generator=torch.Generator().manual_seed(0)) * 3
    hi, lo = S.split(x)
    assert torch.equal(hi, x.to(torch.bfloat16))
    assert torch.equal((x.double() - hi.double()), (x - hi.float()).double())   # the fp32 residual is exact
    assert torch.equal(lo, (x.double() - hi.double()).to(torch.bfloat16))
    assert float(((S.value(hi, lo) - x.double()).abs() / x.double().abs()).max()) <= 2.0 ** -16


@pytest.mark.parametrize("Nf,H,W,C", [(2, 3, 5, 16), (1, 5, 9, 32), (3, 4, 6, 64)])
def test_image_layout_element_by_element(Nf, H, W, C):
    g = torch.Generator().manual_seed(H * W + C)
    x = torch.randn(Nf, H, W, C, generator=g)
    img, lo_off = S.encode(x)
    Hp, Wp, pin, _ = S.geometry(H, W)
    assert lo_off == S.image_elems(Nf, H, W, C) == Nf * C * Hp * Wp + (pin + 8) * 8 and lo_off % 8 == 0
    assert img.numel() == 2 * lo_off
    hi, lo = S.split(x)
    want = torch.zeros(2 * lo_off, dtype=torch.bfloat16)
    for n in range(Nf):
        for y in range(H):
            for xx in range(W):
                for c in range(C):
                    i = ((n * (C // 8) + c // 8) * Hp * Wp + (y + 1) * Wp + (xx + 1)) * 8 + c % 8
                    want[i], want[lo_off + i] = hi[n, y, xx, c], lo[n, y, xx, c]
    assert torch.equal(img.view(torch.int16), want.view(torch.int16))
    assert torch.equal(S.decode(img, lo_off, Nf, H, W, C), S.value(hi, lo))
    dh, dl = S.decode_planes(img, lo_off, Nf, H, W, C)
    assert torch.equal(S.encode_planes(dh, dl)[0].view(torch.int16), img.view(torch.int16))


def test_relu_encoding():
    x = torch.randn(2, 6, 7, 16, generator=torch.Generator().manual_seed(1))
    img, lo_off = S.encode(x, relu=True)
    assert torch.equal(S.decode(img, lo_off, 2, 6, 7, 16), S.value(*S.split(x.clamp_min(0))))


@pytest.mark.parametrize("H,W", [(7, 7), (8, 8), (7, 10), (10, 9), (3, 5), (21, 21)])
def test_maxpool_taps_match_torch_with_ties(H, W):
    g = torch.Generator().manual_seed(H * 31 + W)
    x = torch.randint(-2, 3, (3, H, W, 16), generator=g).float()   # few values: many tied windows
    y, taps = S.maxpool_taps(x)
    ty, idx = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1, return_indices=True)
    assert torch.equal(y, ty.permute(0, 2, 3, 1))
    OH, OW = y.shape[1:3]
    oy = torch.arange(OH).view(1, OH, 1, 1)
    ox = torch.arange(OW).view(1, 1, OW, 1)
    idx = idx.permute(0, 2, 3, 1)
    kh, kw = idx // W - (2 * oy - 1), idx % W - (2 * ox - 1)
    assert torch.equal(taps.long(), kh * 3 + kw)


@pytest.mark.parametrize("H,W", [(7, 7), (8, 10), (11, 6)])
def test_maxpool_scatter_is_the_pool_gradient(H, W):
    g = torch.Generator().manual_seed(H + 5 * W)
    x = torch.randint(-2, 3, (2, H, W, 16), generator=g).double()
    _, taps = S.maxpool_taps(x)
    xr = x.permute(0, 3, 1, 2).clone().requires_grad_(True)
    y = torch.nn.functional.max_pool2d(xr, 3, 2, 1)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    got = S.maxpool_scatter(dy.permute(0, 2, 3, 1), taps, H, W)
    torch.testing.assert_close(got, xr.grad.permute(0, 2, 3, 1), rtol=1e-15, atol=1e-15)


def test_conv_references_are_autograd_of_conv2d():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 6, 9, 16, generator=g, dtype=torch.float64)
    w = torch.randn(32, 16, 3, 3, generator=g, dtype=torch.float64)
    xr, wr = x.permute(0, 3, 1, 2).clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = torch.nn.functional.conv2d(xr, wr, padding=1)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    dyn = dy.permute(0, 2, 3, 1)
    torch.testing.assert_close(S.conv3x3(x, w), y.detach().permute(0, 2, 3, 1))
    torch.testing.assert_close(S.conv3x3_input_grad(dyn, w), xr.grad.permute(0, 2, 3, 1))
    torch.testing.assert_close(S.conv3x3_weight_grad(dyn, x), wr.grad)


@pytest.mark.parametrize("C,O,W", [(16, 16, 5), (64, 32, 21)])
def test_tolerance_admits_split_fp32_and_rejects_a_lost_lo_product(C, O, W):
    """The three products of the split kernels, formed and summed in fp32, stay inside the tolerance; the same float64
    reference without the x_lo.w_hi product is at least ten times outside it."""
    g = torch.Generator().manual_seed(C + O)
    x, w = torch.randn(8, 7, W, C, generator=g), torch.randn(O, C, 3, 3, generator=g) * 0.1
    (xh, xl), (wh, wl) = S.split(x), S.split(w)
    ref = S.conv3x3(S.value(xh, xl), S.value(wh, wl))
    c32 = lambda a, b: S._nhwc(torch.nn.functional.conv2d(S._nchw(a.float()), b.float(), padding=1))
    split32 = c32(xh, wh) + c32(xh, wl) + c32(xl, wh)
    tol = S.tolerance(9 * C, S.rms(S.value(xh, xl)) * S.rms(S.value(wh, wl)), ref)
    assert S.excess(split32, ref, tol) <= 1.0
    assert S.excess(ref - S.conv3x3(xl, wh), ref, tol) >= 10.0


@pytest.mark.parametrize("M,N,K", [(64, 48, 64), (128, 96, 520), (32, 64, 3136), (32, 256, 20000)])
def test_single_plane_tolerance_admits_fp32_sums_and_rejects_a_lost_k_block(M, N, K):
    """lolo=False: bf16 operands multiplied exactly and summed in fp32 stay inside the bound; the float64 reference
    without the products of one 64-term k-block is at least ten times outside it."""
    g = torch.Generator().manual_seed(M + K)
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).double()
    b = (torch.randn(N, K, generator=g) * 0.1).to(torch.bfloat16).double()
    ref = a @ b.t()
    tol = S.tolerance(K, S.rms(a) * S.rms(b), ref, lolo=False)
    assert S.excess(a.float() @ b.float().t(), ref, tol) <= 1.0
    assert S.excess(ref - a[:, :64] @ b[:, :64].t(), ref, tol) >= 10.0
