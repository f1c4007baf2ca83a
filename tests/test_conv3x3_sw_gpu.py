"""GPU: the IMPALA ResNet's shifted-window split-bf16 convolutions (csrc/conv3x3_sw.cu) in isolation, against float64
references on the hi + lo operand values (tests/sw_image.py).

Every buffer a producer or kernel writes is filled with 0xFF bytes (NaN) first, so every element a test reads was
written by that call.  Each convolution case also checks that the float64 reference without one lo product is at least
ten times outside the tolerance: a kernel that lost that product would fail the case.  The forward cases run both
kernels (all weights resident, or the wide kernel that streams the window per k16 step in 32-column blocks), the
smallest images, odd sizes, the widest row each pair fits, and frame counts from one to a learner-size call whose CTAs
walk many tiles, unequal in number."""
import pytest
import torch

from tests import sw_image as S

pytestmark = pytest.mark.gpu

NUM_SMS = 132
SMEM = 227 * 1024
PAIRS = [(ck, no) for ck in (16, 32, 64) for no in (16, 32, 64)]


def resident(H, W, CK, NO):
    """sw_fwd_resident (conv3x3_sw.cu): 16 / 32-channel pairs run on sw_conv_fwd_kernel when its shared memory (weights,
    four whole-window stages, barriers, two staging tiles, static column-sum staging) fits; the rest on the wide kernel."""
    pin = S.geometry(H, W)[2]
    smem = 128 + 2 * 9 * CK * NO * 2 + 4 * 2 * (CK // 8) * pin * 16 + 8 * 10 + 2 * 128 * (NO + 4) * 4 + 16
    return CK <= 32 and NO <= 32 and smem + 4 * 8 * 32 * (NO + 1) <= SMEM


def _lib():
    from torchbeast_b200 import _lib
    return _lib


def nan(n, dtype=torch.float32):
    """n elements of dtype, every byte 0xFF (NaN for fp32 and bf16)."""
    nbytes = n * torch.empty(0, dtype=dtype).element_size()
    return torch.full((nbytes,), 255, dtype=torch.uint8, device="cuda").view(dtype)


def bits(x):
    return x.view(torch.int16)


def pack(w, transpose=0, c_real=0):
    """fp32 weights [O, C', 3, 3] -> the packed operand (NaN-prefilled) and the float64 hi + lo / hi / lo weights."""
    L, p = _lib(), _lib().ptr
    O = w.shape[0]
    C = w.shape[1] if not c_real else 16
    wk = nan(L.lib().tb_sw_weight_elems(O, C), torch.bfloat16)
    L.check(L.lib().tb_sw_pack_weights(p(w), p(wk), O, C, transpose, c_real, L.stream_ptr()), "tb_sw_pack_weights")
    hi, lo = S.split(w)
    return wk, S.value(hi, lo), hi.double(), lo.double()


def image(x):
    """fp32 NHWC -> (image through the helper encoder, lo offset, float64 hi + lo, float64 hi, float64 lo)."""
    hi, lo = S.split(x)
    img, E = S.encode_planes(hi, lo)
    return img, E, S.value(hi, lo), hi.double(), lo.double()


def conv_fwd(img, E, wk, Nf, H, W, CK, NO, scale=1.0, bias=None, mask=None, addend=None, emit=False, emit_relu=0,
             csum=False):
    L, p = _lib(), _lib().ptr
    out = nan(Nf * H * W * NO).view(Nf, H, W, NO)
    em = nan(2 * S.image_elems(Nf, H, W, NO), torch.bfloat16) if emit else None
    rows = L.lib().tb_sw_csum_rows(Nf, H, W)
    cs = nan((rows + 128) * NO) if csum else None
    rc = L.lib().tb_sw_conv_fwd(p(img), E, p(wk), p(out), Nf, H, W, CK, NO, scale, p(bias), p(mask), p(addend), p(em),
                                S.image_elems(Nf, H, W, NO), emit_relu, p(cs), L.stream_ptr())
    L.check(rc, "tb_sw_conv_fwd")
    db = None
    if csum:
        db = nan(NO)
        L.check(L.lib().tb_sw_csum_reduce(p(cs), rows, NO, p(db), L.stream_ptr()), "tb_sw_csum_reduce")
    torch.cuda.synchronize()
    return out, em, db


def check_conv(got, ref, ref_drop, K, scale, extra=None):
    tol = S.tolerance(K, scale, ref, extra=extra)
    assert torch.isfinite(got).all()
    err = S.excess(got, ref, tol)
    assert err <= 1.0, "max |err| / tol = %.3g" % err
    miss = S.excess(ref_drop, ref, tol)
    assert miss >= 10.0, "the reference without a lo product is only %.3g x the tolerance" % miss
    return err


# (CK, NO, H, W, Nf, resident?)
FWD_CASES = [(ck, no, 21, 21, 201, ck <= 32 and no <= 32) for ck, no in PAIRS]   # 804 tiles: CTAs walk unequal counts
FWD_CASES += [
    (16, 16, 3, 5, 1, True), (16, 64, 3, 5, 3, False), (64, 16, 5, 9, 1, False), (32, 32, 5, 9, 3, True),
    (64, 64, 9, 17, 3, False), (32, 16, 9, 17, 1, True), (16, 32, 21, 21, 3, True), (64, 32, 37, 53, 3, False),
    (32, 32, 37, 53, 1, True), (32, 32, 11, 54, 3, False), (32, 32, 84, 84, 3, False), (16, 32, 84, 84, 1, True),
    (16, 16, 126, 126, 3, True), (32, 32, 126, 126, 1, False), (32, 16, 126, 126, 1, False), (64, 64, 7, 101, 3, False),
]


@pytest.mark.parametrize("CK,NO,H,W,Nf,res", FWD_CASES)
def test_forward_vs_fp64(CK, NO, H, W, Nf, res):
    assert resident(H, W, CK, NO) == res
    g = torch.Generator(device="cuda").manual_seed(CK * 7 + NO + H * W + Nf)
    x = torch.randn(Nf, H, W, CK, device="cuda", generator=g)
    w = torch.randn(NO, CK, 3, 3, device="cuda", generator=g) * 0.1
    img, E, xv, xh, xl = image(x)
    wk, wv, wh, _ = pack(w)
    out, _, _ = conv_fwd(img, E, wk, Nf, H, W, CK, NO)
    ref = S.conv3x3(xv, wv)
    check_conv(out, ref, ref - S.conv3x3(xl, wh), 9 * CK, S.rms(xv) * S.rms(wv))


def test_resident_wide_boundary():
    """32 -> 32 runs on the resident kernel up to W = 53 and on the wide kernel from W = 54 (restated rule)."""
    assert resident(8, 53, 32, 32) and not resident(8, 54, 32, 32)
    assert all(not resident(8, 5, ck, no) for ck, no in PAIRS if 64 in (ck, no))


# learner-size calls: every frame is independent, so the first, the last and sampled frames are checked
@pytest.mark.parametrize("CK,NO,H,W,Nf", [(16, 32, 84, 84, 648), (32, 32, 21, 21, 2592), (64, 64, 21, 21, 2592)])
def test_forward_learner_size(CK, NO, H, W, Nf):
    g = torch.Generator(device="cuda").manual_seed(Nf + CK + NO)
    x = torch.randn(Nf, H, W, CK, device="cuda", generator=g)
    w = torch.randn(NO, CK, 3, 3, device="cuda", generator=g) * 0.1
    b = torch.randn(NO, device="cuda", generator=g)
    img, E, xv, xh, xl = image(x)
    del x
    wk, wv, wh, _ = pack(w)
    out, _, _ = conv_fwd(img, E, wk, Nf, H, W, CK, NO, bias=b)
    pick = torch.tensor(sorted({0, 1, Nf // 3, Nf // 2 + 1, Nf - 2, Nf - 1} |
                               set(torch.randint(0, Nf, (10,), generator=g, device="cuda").tolist())), device="cuda")
    ref = S.conv3x3(xv[pick], wv) + b.double()
    check_conv(out[pick], ref, ref - S.conv3x3(xl[pick], wh), 9 * CK, S.rms(xv[pick]) * S.rms(wv), extra=b.double())


@pytest.mark.parametrize("CK,NO,H,W,Nf", [(16, 32, 13, 11, 5), (64, 32, 9, 9, 7), (16, 64, 10, 33, 3)])
def test_epilogue_scale_bias(CK, NO, H, W, Nf):
    g = torch.Generator(device="cuda").manual_seed(CK + NO + W)
    x = torch.randn(Nf, H, W, CK, device="cuda", generator=g)
    w = torch.randn(NO, CK, 3, 3, device="cuda", generator=g) * 0.1
    b = torch.randn(NO, device="cuda", generator=g)
    img, E, xv, xh, xl = image(x)
    wk, wv, wh, _ = pack(w)
    out, _, _ = conv_fwd(img, E, wk, Nf, H, W, CK, NO, scale=0.375, bias=b)
    ref = S.conv3x3(xv, wv) * 0.375 + b.double()
    check_conv(out, ref, ref - 0.375 * S.conv3x3(xl, wh), 9 * CK, 0.375 * S.rms(xv) * S.rms(wv), extra=b.double())


# the input-gradient form: the dY image (O channels) through transposed, flipped weights, the ReLU mask, then the skip
# gradient; emit writes dX as the next conv's dY image and csum its column sums (its bias gradient)
@pytest.mark.parametrize("O,C,H,W,Nf", [(32, 32, 11, 11, 9), (16, 32, 21, 21, 201), (64, 16, 9, 17, 5), (64, 64, 11, 11, 3),
                                        (32, 16, 5, 5, 1)])
def test_input_gradient_mask_addend_emit_csum(O, C, H, W, Nf):
    g = torch.Generator(device="cuda").manual_seed(O * 3 + C + H * W)
    dy = torch.randn(Nf, H, W, O, device="cuda", generator=g)
    w = torch.randn(O, C, 3, 3, device="cuda", generator=g) * 0.1
    mask = torch.randn(Nf, H, W, C, device="cuda", generator=g)
    add = torch.randn(Nf, H, W, C, device="cuda", generator=g)
    img, E, dv, dh, dl = image(dy)
    wk, wv, wh, _ = pack(w, transpose=1)
    out, em, db = conv_fwd(img, E, wk, Nf, H, W, O, C, mask=mask, addend=add, emit=True, csum=True)
    keep = (mask > 0).double()
    ref = S.conv3x3_input_grad(dv, wv) * keep + add.double()
    drop = (S.conv3x3_input_grad(dv, wv) - S.conv3x3_input_grad(dl, wh)) * keep + add.double()
    check_conv(out, ref, drop, 9 * O, S.rms(dv) * S.rms(wv), extra=add.double())
    _check_emit(out, em, 0)
    _check_csum(out, db)


@pytest.mark.parametrize("CK,NO,H,W,Nf,emit_relu", [(32, 32, 11, 11, 7, 1), (16, 64, 9, 9, 3, 1), (64, 16, 13, 7, 5, 0),
                                                    (16, 16, 126, 126, 3, 1), (32, 32, 126, 126, 2, 0),
                                                    (64, 64, 6, 101, 2, 1), (16, 32, 3, 5, 1, 1)])
def test_emit_image_bits(CK, NO, H, W, Nf, emit_relu):
    """The emitted hi / lo image equals, bit for bit and borders and slack included, what sw_pad_split makes from
    relu?(out).  At W = 126 (padded rows of 128 pixels) the first tile's border writes must reach pixel Wp = 128."""
    g = torch.Generator(device="cuda").manual_seed(CK + NO * 5 + W)
    x = torch.randn(Nf, H, W, CK, device="cuda", generator=g)
    w = torch.randn(NO, CK, 3, 3, device="cuda", generator=g) * 0.1
    b = torch.randn(NO, device="cuda", generator=g)
    img, E, xv, xh, xl = image(x)
    wk, wv, wh, _ = pack(w)
    out, em, db = conv_fwd(img, E, wk, Nf, H, W, CK, NO, bias=b, emit=True, emit_relu=emit_relu, csum=True)
    ref = S.conv3x3(xv, wv) + b.double()
    check_conv(out, ref, ref - S.conv3x3(xl, wh), 9 * CK, S.rms(xv) * S.rms(wv), extra=b.double())
    _check_emit(out, em, emit_relu)
    _check_csum(out, db)


def _check_emit(out, em, emit_relu):
    L, p = _lib(), _lib().ptr
    Nf, H, W, C = out.shape
    E = S.image_elems(Nf, H, W, C)
    want = nan(2 * E, torch.bfloat16)
    L.check(L.lib().tb_sw_pad_split_f32(p(out), p(want), E, Nf, H, W, C, emit_relu, None, None, 0, L.stream_ptr()),
            "tb_sw_pad_split_f32")
    torch.cuda.synchronize()
    assert torch.equal(bits(em), bits(want))
    assert torch.equal(bits(em), bits(S.encode(out, relu=bool(emit_relu))[0]))


def _check_csum(out, db):
    """csum + sw_csum_reduce = the column sums of the result over valid pixels only (padding rows must add nothing)."""
    o = out.reshape(-1, out.shape[-1]).double()
    ref = o.sum(0)
    tol = S.tolerance(o.shape[0], S.rms(o), ref)
    assert S.excess(db, ref, tol) <= 1.0


# ---- weight gradient ---------------------------------------------------------------------------------------------
def wgrad(dyimg, dE, ximg, xE, Nf, H, W, C, O, scale=1.0, c_real=0, partial_floats=None):
    L, p = _lib(), _lib().ptr
    dw = nan(O * (c_real or C) * 9).view(O, c_real or C, 3, 3)
    n = NUM_SMS * O * 9 * C if partial_floats is None else partial_floats
    part = nan(n)
    rc = L.lib().tb_sw_conv_wgrad(p(dyimg), dE, p(ximg), xE, p(dw), Nf, H, W, C, O, scale, c_real, p(part), n,
                                  L.stream_ptr())
    return rc, dw


WGRAD_CASES = [(c, o, 13, 13, 5) for c, o in PAIRS]   # (C, O, H, W, Nf)
WGRAD_CASES += [(32, 16, 7, 5, 9), (64, 64, 5, 5, 3), (32, 64, 21, 21, 648), (16, 16, 84, 84, 20)]


@pytest.mark.parametrize("C,O,H,W,Nf", WGRAD_CASES)
def test_weight_gradient_vs_fp64(C, O, H, W, Nf):
    g = torch.Generator(device="cuda").manual_seed(C * 5 + O + H * W + Nf)
    dy = torch.randn(Nf, H, W, O, device="cuda", generator=g)
    x = torch.randn(Nf, H, W, C, device="cuda", generator=g)
    dimg, dE, dv, dh, dl = image(dy)
    ximg, xE, xv, xh, xl = image(x)
    rc, dw = wgrad(dimg, dE, ximg, xE, Nf, H, W, C, O)
    _lib().check(rc, "tb_sw_conv_wgrad")
    torch.cuda.synchronize()
    ref = S.conv3x3_weight_grad(dv, xv)
    check_conv(dw, ref, ref - S.conv3x3_weight_grad(dl, xh), Nf * H * W, S.rms(dv) * S.rms(xv))


@pytest.mark.parametrize("Cf,O,H,W,Nf", [(4, 16, 21, 21, 40), (3, 32, 9, 33, 7), (12, 64, 11, 11, 5), (1, 16, 5, 5, 3)])
def test_first_conv_forward_and_weight_gradient(Cf, O, H, W, Nf):
    """The first conv of the net: uint8 frames as a 16-channel image (no lo plane), weights with c_real = Cf input
    channels, 1/255 in the forward epilogue and in the weight gradient's scale."""
    L, p = _lib(), _lib().ptr
    g = torch.Generator(device="cuda").manual_seed(Cf + O + W)
    fr = torch.randint(0, 256, (Nf, Cf, H, W), dtype=torch.uint8, device="cuda", generator=g)
    w = torch.randn(O, Cf, 3, 3, device="cuda", generator=g) * 0.1
    b = torch.randn(O, device="cuda", generator=g)
    E = S.image_elems(Nf, H, W, 16)
    ximg = nan(2 * E, torch.bfloat16)
    L.check(L.lib().tb_sw_frames_u8(p(fr), p(ximg), E, Nf, Cf, H, W, L.stream_ptr()), "tb_sw_frames_u8")
    wk, wv, wh, wl = pack(w, c_real=Cf)
    out, _, _ = conv_fwd(ximg, E, wk, Nf, H, W, 16, O, scale=1 / 255, bias=b)
    pix = fr.permute(0, 2, 3, 1).double()
    ref = S.conv3x3(pix, wv) / 255 + b.double()
    # the pixels have no lo plane: the product that can be lost is pixel . w_lo
    check_conv(out, ref, ref - S.conv3x3(pix, wl) / 255, 9 * Cf, S.rms(pix) * S.rms(wv) / 255, extra=b.double())

    dy = torch.randn(Nf, H, W, O, device="cuda", generator=g)
    dimg, dE, dv, dh, dl = image(dy)
    rc, dw = wgrad(dimg, dE, ximg, E, Nf, H, W, 16, O, scale=1 / 255, c_real=Cf)
    L.check(rc, "tb_sw_conv_wgrad")
    torch.cuda.synchronize()
    ref = S.conv3x3_weight_grad(dv, pix) / 255
    check_conv(dw, ref, ref - S.conv3x3_weight_grad(dl, pix) / 255, Nf * H * W, S.rms(dv) * S.rms(pix) / 255)


# ---- producers ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,H,W,Nf,relu", [(16, 5, 9, 3, 0), (32, 21, 21, 7, 1), (64, 11, 13, 2, 0), (16, 84, 84, 2, 1),
                                           (32, 3, 126, 1, 0)])
def test_pad_split_bits_and_colsum(C, H, W, Nf, relu):
    L, p = _lib(), _lib().ptr
    g = torch.Generator(device="cuda").manual_seed(C + H + W + relu)
    x = torch.randn(Nf, H, W, C, device="cuda", generator=g)
    E = S.image_elems(Nf, H, W, C)
    img = nan(2 * E, torch.bfloat16)
    L.check(L.lib().tb_sw_pad_split_f32(p(x), p(img), E, Nf, H, W, C, relu, None, None, 0, L.stream_ptr()), "pad_split")
    torch.cuda.synchronize()
    assert torch.equal(bits(img), bits(S.encode(x, relu=bool(relu))[0]))
    # the column-sum form (dY of a conv -> its image and its bias gradient; no ReLU)
    img2, db = nan(2 * E, torch.bfloat16), nan(C)
    n = L.lib().tb_sw_colsum_scratch_floats(Nf, H, W, C)
    scratch = nan(n)
    L.check(L.lib().tb_sw_pad_split_f32(p(x), p(img2), E, Nf, H, W, C, 0, p(db), p(scratch), n, L.stream_ptr()),
            "pad_split_colsum")
    torch.cuda.synchronize()
    assert torch.equal(bits(img2), bits(S.encode(x)[0]))
    ref = x.double().reshape(-1, C).sum(0)
    assert S.excess(db, ref, S.tolerance(Nf * H * W, S.rms(x), ref)) <= 1.0


@pytest.mark.parametrize("Cf", [1, 3, 4, 12, 16])
def test_frames_u8_bits(Cf):
    L, p = _lib(), _lib().ptr
    Nf, H, W = 5, 13, 17
    fr = torch.randint(0, 256, (Nf, Cf, H, W), dtype=torch.uint8, device="cuda",
                       generator=torch.Generator(device="cuda").manual_seed(Cf))
    E = S.image_elems(Nf, H, W, 16)
    img = nan(2 * E, torch.bfloat16)
    L.check(L.lib().tb_sw_frames_u8(p(fr), p(img), E, Nf, Cf, H, W, L.stream_ptr()), "tb_sw_frames_u8")
    torch.cuda.synchronize()
    hi = torch.zeros(Nf, H, W, 16, dtype=torch.bfloat16, device="cuda")
    hi[..., :Cf] = fr.permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(bits(img), bits(S.encode_planes(hi, torch.zeros_like(hi))[0]))


def maxpool(x):
    L, p = _lib(), _lib().ptr
    Nf, H, W, C = x.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y, arg = nan(Nf * OH * OW * C).view(Nf, OH, OW, C), nan(Nf * OH * OW * C, torch.uint8).view(Nf, OH, OW, C)
    L.check(L.lib().tb_maxpool3x3s2_fwd_f32(p(x), p(y), p(arg), Nf, H, W, C, L.stream_ptr()), "tb_maxpool3x3s2_fwd_f32")
    torch.cuda.synchronize()
    return y, arg


@pytest.mark.parametrize("C,H,W,Nf", [(16, 84, 84, 3), (32, 21, 21, 5), (64, 11, 10, 4), (16, 8, 13, 2), (32, 3, 5, 1)])
def test_maxpool_forward_taps_bits(C, H, W, Nf):
    g = torch.Generator(device="cuda").manual_seed(C + H * W)
    x = torch.randint(-2, 3, (Nf, H, W, C), device="cuda", generator=g).float()   # integer values: tied windows
    y, arg = maxpool(x)
    wy, wt = S.maxpool_taps(x)
    assert torch.equal(y, wy) and torch.equal(arg, wt)
    ty = torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(y, ty)


@pytest.mark.parametrize("C,H,W,Nf", [(16, 84, 84, 3), (32, 21, 21, 9), (64, 11, 10, 4), (16, 7, 13, 2), (32, 3, 5, 1)])
def test_pool_backward_image_colsum(C, H, W, Nf):
    L, p = _lib(), _lib().ptr
    g = torch.Generator(device="cuda").manual_seed(C * 3 + H * W)
    x = torch.randint(-2, 3, (Nf, H, W, C), device="cuda", generator=g).float()
    _, arg = maxpool(x)
    OH, OW = arg.shape[1:3]
    dyp = torch.randn(Nf, OH, OW, C, device="cuda", generator=g)
    E = S.image_elems(Nf, H, W, C)
    img, db = nan(2 * E, torch.bfloat16), nan(C)
    n = L.lib().tb_sw_colsum_scratch_floats(Nf, H, W, C)
    scratch = nan(n)
    L.check(L.lib().tb_sw_pool_bwd_image_colsum(p(arg), p(dyp), p(img), E, Nf, H, W, C, p(db), p(scratch), n,
                                                L.stream_ptr()), "tb_sw_pool_bwd_image_colsum")
    torch.cuda.synchronize()
    ref = S.maxpool_scatter(dyp, arg, H, W)
    mag = S.maxpool_scatter(dyp.abs(), arg, H, W)
    hi, lo = S.decode_planes(img, E, Nf, H, W, C)
    # at most 4 fp32 additions, then the hi / lo split (2^-16 of the value)
    assert S.excess(S.value(hi, lo), ref, 2.0 ** -15 * mag + 1e-30) <= 1.0
    assert torch.equal(bits(img), bits(S.encode_planes(hi, lo)[0]))   # borders and slack zero
    cref = ref.reshape(-1, C).sum(0)
    assert S.excess(db, cref, S.tolerance(Nf * H * W, S.rms(ref), cref, extra=mag.reshape(-1, C).sum(0))) <= 1.0


# ---- host-side rejections: an error before any launch ------------------------------------------------------------
def test_host_rejections():
    L, p = _lib(), _lib().ptr
    h = L.lib()
    Nf, H = 2, 5
    img = torch.zeros(2 * S.image_elems(Nf, H, 102, 64), dtype=torch.bfloat16, device="cuda")
    wk = torch.zeros(h.tb_sw_weight_elems(64, 64), dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(Nf * H * 102 * 64, device="cuda")
    E = S.image_elems(Nf, H, 102, 64)
    torch.cuda.synchronize()
    n0 = h.tb_launch_count()
    rc = h.tb_sw_conv_fwd(p(img), E, p(wk), p(out), Nf, H, 102, 64, 64, 1.0, None, None, None, None, 0, 0, None,
                          L.stream_ptr())
    assert rc != 0 and b"unsupported shape" in h.tb_last_error()
    assert h.tb_launch_count() == n0   # (W = 101, the widest row 64 -> 64 fits, runs in test_forward_vs_fp64)

    E4 = S.image_elems(Nf, H, 4, 32)
    i4 = torch.zeros(2 * E4, dtype=torch.bfloat16, device="cuda")
    rc, _ = wgrad(i4, E4, i4, E4, Nf, H, 4, 32, 32)
    assert rc != 0 and b"W = 4 < 5" in h.tb_last_error()
    E5 = S.image_elems(Nf, H, 5, 32)
    i5 = torch.zeros(2 * E5, dtype=torch.bfloat16, device="cuda")
    tiles = Nf * S.geometry(H, 5)[3]
    need = min(NUM_SMS, tiles) * 32 * 9 * 32
    n1 = h.tb_launch_count()
    rc, _ = wgrad(i5, E5, i5, E5, Nf, H, 5, 32, 32, partial_floats=need - 1)
    assert rc != 0 and b"partial buffer too small" in h.tb_last_error()
    assert h.tb_launch_count() == n1
    rc, _ = wgrad(i5, E5, i5, E5, Nf, H, 5, 32, 32, partial_floats=need)
    assert rc == 0
    torch.cuda.synchronize()
