"""Plain-torch restatement of the split-bf16 convolution formats and their float64 references (no kernels here).

- The padded planar image of the ResNet shifted-window convolutions (csrc/conv3x3_sw.cuh): one plane of
  [Nf][C/8][(H+2)*(W+2)][8] bf16 elements (frame, 8-channel chunk, zero-padded pixel, channel in the chunk) followed by
  zero slack that a frame's last 128-pixel tile reads past the last plane; the lo plane follows at lo_off elements.
- The split of an fp32 value into hi = RNE bf16(x) and lo = RNE bf16(x - hi), as split_bf16x2 does (x - hi is exact).
- The argmax taps of nn.MaxPool2d(3, 2, 1): kh*3 + kw of each window's first maximum in row-major tap order.
- float64 3x3 / stride 1 / pad 1 convolution, input gradient and weight gradient of NHWC tensors.
- The tolerance of a split-bf16 product against a float64 reference on the same hi + lo operand values.

Every function works on any device, so tests/test_conv3x3_sw_cpu.py checks them without a GPU."""
import torch
import torch.nn.functional as F

TILE = 128           # output pixels per tile of the shifted-window kernels
U_BF16 = 2.0 ** -8   # unit roundoff of bf16 (8 significant bits)
U_F32 = 2.0 ** -24   # unit roundoff of fp32


def geometry(H, W):
    """(Hp, Wp, pin, tiles per frame) as sw_geom computes them: pin = pixels of a tile's input window."""
    Hp, Wp = H + 2, W + 2
    pin = (TILE + 2 * Wp + 2 + 7) & ~7
    vend = (H - 1) * Wp + W
    return Hp, Wp, pin, -(-vend // TILE)


def image_elems(Nf, H, W, C):
    """Elements of one plane of the padded planar image, slack included (sw_image_elems)."""
    Hp, Wp, pin, _ = geometry(H, W)
    return Nf * (C // 8) * Hp * Wp * 8 + (pin + 8) * 8


def split(x):
    """fp32 -> (hi, lo) bf16 with hi = RNE(x), lo = RNE(x - hi)."""
    x = x.float()
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def value(hi, lo):
    """float64 value hi + lo of a split operand."""
    return hi.double() + lo.double()


def encode_planes(hi, lo):
    """bf16 NHWC hi / lo [Nf, H, W, C] -> bf16 [2 * E] padded planar image (hi plane, lo plane at E), borders and slack
    zero; returns (image, E)."""
    Nf, H, W, C = hi.shape
    E = image_elems(Nf, H, W, C)
    img = torch.zeros(2, E, dtype=torch.bfloat16, device=hi.device)
    body = Nf * C * (H + 2) * (W + 2)
    for pl, v in enumerate((hi, lo)):
        pad = F.pad(v, (0, 0, 1, 1, 1, 1))
        img[pl, :body] = pad.reshape(Nf, H + 2, W + 2, C // 8, 8).permute(0, 3, 1, 2, 4).reshape(-1)
    return img.reshape(-1), E


def encode(x, relu=False):
    """fp32 NHWC [Nf, H, W, C] (through ReLU if relu) -> (padded planar hi / lo image, lo offset), as sw_pad_split."""
    return encode_planes(*split(x.clamp_min(0) if relu else x))


def decode_planes(img, lo_off, Nf, H, W, C):
    """Inverse of encode_planes: (hi, lo) bf16 NHWC of the interior pixels."""
    body = Nf * C * (H + 2) * (W + 2)
    out = []
    for base in (0, lo_off):
        v = img[base:base + body].reshape(Nf, C // 8, H + 2, W + 2, 8).permute(0, 2, 3, 1, 4).reshape(Nf, H + 2, W + 2, C)
        out.append(v[:, 1:H + 1, 1:W + 1])
    return tuple(out)


def decode(img, lo_off, Nf, H, W, C):
    """float64 NHWC hi + lo of the interior pixels of an image."""
    return value(*decode_planes(img, lo_off, Nf, H, W, C))


def maxpool_taps(x):
    """nn.MaxPool2d(3, 2, 1) on NHWC x -> (y, taps uint8): taps = kh*3 + kw of each window's first maximum."""
    Nf, H, W, C = x.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(x, (0, 0, 1, 1, 1, 1), value=float("-inf"))
    best = torch.full((Nf, OH, OW, C), float("-inf"), dtype=x.dtype, device=x.device)
    taps = torch.zeros(Nf, OH, OW, C, dtype=torch.uint8, device=x.device)
    for kh in range(3):
        for kw in range(3):
            v = xp[:, kh:kh + 2 * OH - 1:2, kw:kw + 2 * OW - 1:2]
            better = v > best
            best = torch.where(better, v, best)
            taps = torch.where(better, torch.full_like(taps, kh * 3 + kw), taps)
    return best, taps


def maxpool_scatter(dy, taps, H, W):
    """float64 gradient of nn.MaxPool2d(3, 2, 1) through recorded taps: dy [Nf, OH, OW, C] -> dx [Nf, H, W, C]."""
    Nf, OH, OW, C = dy.shape
    dxp = torch.zeros(Nf, H + 2, W + 2, C, dtype=torch.float64, device=dy.device)
    for kh in range(3):
        for kw in range(3):
            hit = (taps == kh * 3 + kw).double() * dy.double()
            dxp[:, kh:kh + 2 * OH - 1:2, kw:kw + 2 * OW - 1:2] += hit
    return dxp[:, 1:H + 1, 1:W + 1]


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def conv3x3(x, w):
    """float64 3x3 / stride 1 / pad 1 convolution: x NHWC [Nf, H, W, C], w [O, C, 3, 3] -> NHWC [Nf, H, W, O]."""
    return _nhwc(F.conv2d(_nchw(x.double()), w.double(), padding=1))


def conv3x3_input_grad(dy, w):
    """float64 input gradient of conv3x3: dy NHWC [Nf, H, W, O] -> NHWC [Nf, H, W, C]."""
    Nf, H, W, _ = dy.shape
    return _nhwc(torch.nn.grad.conv2d_input((Nf, w.shape[1], H, W), w.double(), _nchw(dy.double()), padding=1))


def conv3x3_weight_grad(dy, x):
    """float64 weight gradient of conv3x3: dy NHWC [Nf, H, W, O], x NHWC [Nf, H, W, C] -> [O, C, 3, 3]."""
    return torch.nn.grad.conv2d_weight(_nchw(x.double()), (dy.shape[3], x.shape[3], 3, 3), _nchw(dy.double()), padding=1)


def rms(x):
    return float(x.double().pow(2).mean().sqrt())


def tolerance(K, scale, ref, rtol=2.0 ** -20, extra=None, lolo=True):
    """Bound on |split-bf16 result - float64 reference on the hi + lo operands| for sums of K products of RMS size
    `scale` (epilogue scale factor included).  Operands are exact as hi + lo, so the error has two sources:
      - the lo.lo product the kernels never issue: |x_lo w_lo| <= u^2 |x| |w| with u = 2^-8 per product;
      - fp32 accumulation, at most 2^-24 of the running sum per addition, taken over a chain of all K terms.
    Both add K terms of independent sign, so their spread is sqrt(K) * scale * (u^2 + 2^-24 sqrt(K)); the bound allows six
    times that, plus rtol of the magnitude of the result (and of `extra`, e.g. a residual addend) for the epilogue's
    fp32 roundings.  An operand whose lo plane is dropped moves a result by about 2^-9 sqrt(K) scale, far outside it.
    lolo=False: single-plane bf16 operands against the float64 product of those same bf16 values.  No lo.lo term exists
    and fp32 accumulation is the only source, so it is charged as the tensor cores do it: they add each group of 16
    products to the running sum with truncation, not rounding (Fasi et al., "Numerical behavior of NVIDIA tensor
    cores", PeerJ CS 2021), so each of the K/16 additions loses about 2^-24 of the sum in the same direction and the
    losses add up instead of cancelling: (K/16) 2^-24 sqrt(K) scale, where that exceeds the rounding term (K > 256).
    On an H100 (700 W) the rounding term alone was exceeded 1.87 times at K = 20000.  A 64-term k-block left out moves
    a result by about 8 scale, far outside it."""
    acc = U_F32 * (K ** 0.5 if lolo else max(K ** 0.5, K / 16.0))
    tol = 6.0 * scale * K ** 0.5 * ((U_BF16 ** 2 if lolo else 0.0) + acc) + rtol * ref.abs()
    return tol if extra is None else tol + rtol * extra.abs()


def excess(got, ref, tol):
    """max |got - ref| / tol (<= 1 passes)."""
    return float(((got.double() - ref).abs() / tol).max())
