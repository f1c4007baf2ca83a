"""GPU: the AtariNet trunk convolutions of the split-bf16 (bf16x3, default) backend in isolation, against float64 torch on
the hi + lo operand values: conv_tc_kernel<..., SPLIT = true> (conv2 / conv3 forward and input gradient),
conv_wgrad_implicit_kernel<3 | 2, true> and the split conv1 over uint8 frames, at the frame counts of
test_trunk_tiles_gpu.py (one frame up to the learner's 2592, with partial last tiles and stages).

Outputs are prefilled with 0xFF bytes (NaN).  The tolerance is tests/sw_image.py's; every case also checks that the
float64 reference without one lo product (the A operand's lo plane times the B operand's hi plane; for conv1, whose pixels
have no lo plane, the weights' lo plane) is at least ten times outside it."""
import pytest
import torch

from tests import sw_image as S

pytestmark = pytest.mark.gpu

NUM_SMS = 132
CONVS = [  # H, W, C, K, S, O
    (20, 20, 32, 4, 2, 64),   # conv2: 81 patches per frame, input gradient in 4 parity classes of 100 pixels
    (9, 9, 64, 3, 1, 64),     # conv3: 49 patches per frame, input gradient over 81 pixels
]
FRAMES = [1, 2, 7, 2591, 2592]


def _lib():
    from torchbeast_b200 import _lib
    return _lib


def nan(n, dtype=torch.float32):
    nbytes = n * torch.empty(0, dtype=dtype).element_size()
    return torch.full((nbytes,), 255, dtype=torch.uint8, device="cuda").view(dtype)


def planes(x):
    """fp32 tensor -> (bf16 [2, numel] hi / lo planes, lo offset, float64 hi + lo, float64 hi, float64 lo)."""
    hi, lo = S.split(x)
    return torch.stack([hi.reshape(-1), lo.reshape(-1)]), x.numel(), S.value(hi, lo), hi.double(), lo.double()


def hilo(buf, shape):
    return S.value(buf[0].view(shape), buf[1].view(shape))


def nchw(x):
    return x.permute(0, 3, 1, 2)


def nhwc(x):
    return x.permute(0, 2, 3, 1)


def wgrad_stages(OH, OW):
    """conv_tc_wgrad_implicit: whole frames per stage (rows = patches, padded to 16); the split ring holds 6 operand
    groups per stage and takes 3 stages when they fit, else 2."""
    rows = OH * OW * min(128 // (OH * OW), 256)
    rows_pad = (rows + 15) // 16 * 16
    return 3 if 3 * 6 * rows_pad * 128 + 2048 <= 227 * 1024 else 2


def check(got, ref, ref_drop, K, scale, rtol=2.0 ** -20, extra=None):
    tol = S.tolerance(K, scale, ref, rtol=rtol, extra=extra)
    assert torch.isfinite(got).all()
    err = S.excess(got, ref, tol)
    assert err <= 1.0, "max |err| / tol = %.3g" % err
    miss = S.excess(ref_drop, ref, tol)
    assert miss >= 10.0, "the reference without a lo product is only %.3g x the tolerance" % miss


# the hi + lo planes of a bf16 output carry the fp32 value to 2^-16 of itself
OUT_RTOL = 2.0 ** -16 + 2.0 ** -20

# bf16 bit patterns of ReLU-mask values the input gradient must zero (NaN of either sign and a signalling one, +0, -0, a
# negative subnormal) or keep (the smallest positive subnormal)
MASK_EDGES = [0x7FC0, 0xFFC0, 0x7F81, 0x0000, 0x8000, 0x0001, 0x8001]


def plant_mask_edges(act):
    """every 6th element of the hi plane act[0] replaced by the MASK_EDGES values in turn; returns the plane in float64"""
    edges = torch.tensor([b - (1 << 16) if b >= 1 << 15 else b for b in MASK_EDGES], dtype=torch.int16)
    hi = act[0]
    n = hi[::6].numel()
    hi[::6] = edges.view(torch.bfloat16).to(hi.device).repeat(-(-n // len(MASK_EDGES)))[:n]
    return hi.double()


@pytest.mark.parametrize("H,W,C,K,S_,O", CONVS)
@pytest.mark.parametrize("N", FRAMES)
def test_forward(H, W, C, K, S_, O, N):
    L, p = _lib(), _lib().ptr
    g = torch.Generator(device="cuda").manual_seed(3 * N + H)
    act, a_lo, av, ah, al = planes(torch.randn(N, H, W, C, device="cuda", generator=g))
    w = torch.randn(O, C, K, K, device="cuda", generator=g) * 0.1
    b = torch.randn(O, device="cuda", generator=g)
    OH = (H - K) // S_ + 1
    out = nan(2 * N * OH * OH * O, torch.bfloat16).view(2, -1)
    pack = nan(2 * O * C * K * K, torch.bfloat16)
    L.check(L.lib().tb_conv_nhwc_bf16x3_fwd(p(act), a_lo, p(w), p(b), N, H, W, C, K, K, S_, O, 1, p(out), N * OH * OH * O,
                                            p(pack), L.stream_ptr()), "tb_conv_nhwc_bf16x3_fwd")
    torch.cuda.synchronize()
    wv, wh = S.value(*S.split(w)), S.split(w)[0].double()
    shape = (N, H, W, C)
    pre = nhwc(torch.nn.functional.conv2d(nchw(av.view(shape)), wv, b.double(), stride=S_))
    lost = nhwc(torch.nn.functional.conv2d(nchw(al.view(shape)), wh, stride=S_))
    check(hilo(out, (N, OH, OH, O)), pre.relu(), (pre - lost).relu(), K * K * C, S.rms(av) * S.rms(wv), OUT_RTOL,
          extra=b.double())


@pytest.mark.parametrize("H,W,C,K,S_,O", CONVS)
@pytest.mark.parametrize("N", FRAMES)
def test_input_gradient(H, W, C, K, S_, O, N):
    """Stride 2 (conv2) runs the parity-class path, stride 1 (conv3) the plain one; the ReLU mask is the act hi plane,
    which holds NaN of both signs, +-0 and subnormals (MASK_EDGES): an element is kept exactly where the mask is > 0."""
    L, p = _lib(), _lib().ptr
    g = torch.Generator(device="cuda").manual_seed(5 * N + H)
    OH = (H - K) // S_ + 1
    act, a_lo, _, _, _ = planes(torch.randn(N, H, W, C, device="cuda", generator=g))
    ah = plant_mask_edges(act)
    dy, d_lo, dv, dh, dl = planes(torch.randn(N, OH, OH, O, device="cuda", generator=g))
    w = torch.randn(O, C, K, K, device="cuda", generator=g) * 0.1
    dx = nan(2 * N * H * W * C, torch.bfloat16).view(2, -1)
    pack = nan(2 * O * C * K * K, torch.bfloat16)
    L.check(L.lib().tb_conv_nhwc_bf16x3_dgrad(p(dy), d_lo, p(w), p(act), N, H, W, C, K, K, S_, O, p(dx), N * H * W * C,
                                              p(pack), L.stream_ptr()), "tb_conv_nhwc_bf16x3_dgrad")
    torch.cuda.synchronize()
    wv, wh = S.value(*S.split(w)), S.split(w)[0].double()
    dshape = (N, OH, OH, O)
    keep = (ah.view(N, H, W, C) > 0).double()
    grad = lambda d, ww: nhwc(torch.nn.grad.conv2d_input((N, C, H, W), ww, nchw(d.view(dshape)), stride=S_))
    ref = grad(dv, wv) * keep
    check(hilo(dx, (N, H, W, C)), ref, ref - grad(dl, wh) * keep, K * K * O, S.rms(dv) * S.rms(wv), OUT_RTOL)


@pytest.mark.parametrize("H,W,C,K,S_,O,stages", [c + (st,) for c, st in zip(CONVS, (3, 2))])
@pytest.mark.parametrize("N", FRAMES)
def test_weight_gradient(H, W, C, K, S_, O, stages, N):
    """conv2's 81-patch stages run the 3-stage split ring, conv3's 98-patch stages (two frames) the 2-stage one."""
    OH = (H - K) // S_ + 1
    assert wgrad_stages(OH, OH) == stages
    L, p = _lib(), _lib().ptr
    g = torch.Generator(device="cuda").manual_seed(11 * N + H)
    act, a_lo, av, ah, al = planes(torch.randn(N, H, W, C, device="cuda", generator=g))
    dy, d_lo, dv, dh, dl = planes(torch.randn(N, OH, OH, O, device="cuda", generator=g))
    dw = nan(O * C * K * K).view(O, C, K, K)
    part = nan(NUM_SMS * O * C * K * K)
    L.check(L.lib().tb_conv_nhwc_bf16x3_wgrad(p(dy), d_lo, p(act), a_lo, N, H, W, C, K, K, S_, O, p(dw), p(part),
                                              part.numel(), L.stream_ptr()), "tb_conv_nhwc_bf16x3_wgrad")
    torch.cuda.synchronize()
    grad = lambda d, a: torch.nn.grad.conv2d_weight(nchw(a.view(N, H, W, C)), (O, C, K, K), nchw(d.view(N, OH, OH, O)),
                                                    stride=S_)
    ref = grad(dv, av)
    check(dw, ref, ref - grad(dl, ah), N * OH * OH, S.rms(dv) * S.rms(av))


@pytest.mark.parametrize("N", [1, 7, 2592])
def test_conv1_forward_and_weight_gradient(N):
    """conv1 (8x8, stride 4, 4 -> 32 channels) from uint8 frames: the pixels are exact in bf16, the weights and the
    output (and dY in the weight gradient) have lo planes; 1/255 in the epilogue and in the weight gradient."""
    L, p = _lib(), _lib().ptr
    H = W = 84
    OH = 20
    g = torch.Generator(device="cuda").manual_seed(N + 17)
    fr = torch.randint(0, 256, (N, 4, H, W), dtype=torch.uint8, device="cuda", generator=g)
    w = torch.randn(32, 4, 8, 8, device="cuda", generator=g) * 0.05
    b = torch.randn(32, device="cuda", generator=g)
    out = nan(2 * N * OH * OH * 32, torch.bfloat16).view(2, -1)
    image = nan(N * 4 * H * W, torch.bfloat16)
    pack = nan(2 * 32 * 256, torch.bfloat16)
    L.check(L.lib().tb_conv1_u8_bf16x3_fwd(p(fr), p(w), p(b), N, H, W, 4, 1, p(out), N * OH * OH * 32, p(image), p(pack),
                                           L.stream_ptr()), "tb_conv1_u8_bf16x3_fwd")
    torch.cuda.synchronize()
    pix = fr.double()
    (wh, wl) = (t.double() for t in S.split(w))
    pre = nhwc(torch.nn.functional.conv2d(pix, wh + wl, stride=4)) / 255 + b.double()
    lost = nhwc(torch.nn.functional.conv2d(pix, wl, stride=4)) / 255
    check(hilo(out, (N, OH, OH, 32)), pre.relu(), (pre - lost).relu(), 256, S.rms(pix) * S.rms(wh + wl) / 255, OUT_RTOL,
          extra=b.double())

    dy, d_lo, dv, dh, dl = planes(torch.randn(N, OH, OH, 32, device="cuda", generator=g))
    dw = nan(32 * 4 * 8 * 8).view(32, 4, 8, 8)
    part = nan(NUM_SMS * 32 * 256)
    L.check(L.lib().tb_conv1_u8_bf16x3_wgrad(p(dy), d_lo, p(image), N, H, W, 4, p(dw), p(part), part.numel(),
                                             L.stream_ptr()), "tb_conv1_u8_bf16x3_wgrad")
    torch.cuda.synchronize()
    grad = lambda d: torch.nn.grad.conv2d_weight(pix, (32, 4, 8, 8), nchw(d.view(N, OH, OH, 32)), stride=4) / 255
    ref = grad(dv)
    check(dw, ref, ref - grad(dl), N * OH * OH, S.rms(dv) * S.rms(pix) / 255)
