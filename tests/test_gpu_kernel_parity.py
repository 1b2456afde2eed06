"""Kernel-level parity: every conv kernel variant of the inference path (generic implicit-GEMM kernel, its two-M-tile
form, its staged TMA epilogue, the patch kernel, the K-folded first layers, the fused 4-phase transposed conv) in every
precision, against a float64 reference that rounds where the kernels round.

Reference (float64, torch, on the GPU; float64 never takes the TF32 path):
  F16 / BF16  x^ = round16(x), w^ = round16(w), z = conv(x^, w^),
              y  = round16(act(scale*z + shift [+ x^ for a residual]))
  F32X        the same on the unrounded fp32 operands, no output rounding
round16 is round-to-nearest-even to the context's 16-bit type; scale/shift fold BatchNorm as fold_bn_kernel does
(conv bias into the shift, eps 1e-5).

Bars, derived rather than fitted, with mag = |scale|*conv(|x^|,|w^|) + |shift| + |res| per output element:
  F16 / BF16  |y - ref| <= ulp16(max(|y|,|ref|)) + 2^-16 * mag     (one rounding flip + fp32 accumulation)
              and, with >= 1e4 outputs, |mean(sign(ref) * (y - ref) / ulp16(ref))| <= 0.05 over the elements with
              |ref| > 2^-16 * mag (a truncating conversion gives about -0.5; elements within the accumulation error
              of zero are left out because a ReLU can move them by a whole value, not by a rounding step)
  F32X        |y - ref| <= 2^-15 * mag + lo_step(max(|y|,|ref|))     (split operands carry ~22 bits: about 2^-16 is
              expected, a dropped x_lo*w_hi / x_hi*w_lo pass or residual lo plane costs about 2^-12; lo_step is the
              rounding of the fp16 lo plane, ~2^-22 |y|, down to 2^-25 absolute where lo is subnormal)
Every case also runs twice (bit-identical: inference has no atomics), leaves the fp16 range flag clear, and asserts
the kernel family / BN / BK / MT / staged epilogue / fold that w2l_debug_plan_kernels reports for it.  The S3FD cases use
its conv + ReLU and plain (no activation) kinds, which have no BatchNorm: scale 1, shift = conv bias.

Measured on one H100 SXM (80 GB, 700 W).  Values near 1 in F16 / BF16 are single last-bit flips where the
accumulation term is small; the largest |bias| over all cases was 0.008 ulp; F32X reaches at most 0.06 of its bar except
on fc6 (0.48: its border outputs are the bias alone, bounded by the lo-plane term).
max err/bar in F16 and BF16 (default and generic-only dispatch), and in F32X err/bar and err/mag:
  case                                                  f16  bf16  f32x    err/mag
  gen 7x7 6->16 96x96                                  0.91  0.98  0.033  1.0e-06
  gen 16->32 s2 96x96                                  0.89  0.98  0.015  4.7e-07
  gen 32 res 48x48                                     0.94  0.65  0.019  5.9e-07
  gen 32->64 s2 48x48                                  0.91  0.06  0.019  5.8e-07
  gen 64 res 24x24                                     0.90  0.96  0.022  6.6e-07
  gen 64->128 s2 24x24                                 0.88  0.96  0.021  6.5e-07
  gen 128 res 12x12                                    0.88  0.94  0.027  8.3e-07
  gen 128->256 s2 12x12                                0.77  0.85  0.027  8.4e-07
  gen 256 res 6x6                                      0.85  0.94  0.032  9.9e-07
  gen 256->512 s2 6x6                                  0.69  0.96  0.033  1.0e-06
  gen 512 res 3x3                                      0.79  0.91  0.039  1.2e-06
  gen 512 3x3 pad0 -> 1x1                              0.43  0.02  0.039  1.2e-06
  gen 512 1x1                                          0.30  0.00  0.024  7.2e-07
  audio 1->32 80x16                                    0.97  0.00  0.029  8.8e-07
  audio 32 res 80x16                                   0.90  0.99  0.019  5.8e-07
  audio 32->64 s(3,1)                                  0.89  0.95  0.016  5.0e-07
  audio 64 res 27x16                                   0.87  0.99  0.019  5.8e-07
  audio 64->128 s3                                     0.89  0.97  0.019  5.8e-07
  audio 128 res 9x6                                    0.91  0.94  0.023  6.9e-07
  audio 128->256 s(3,2)                                0.35  0.08  0.022  6.6e-07
  audio 256 res 3x3                                    0.86  0.97  0.030  9.1e-07
  audio 256->512 3x3 pad0                              0.50  0.00  0.025  7.5e-07
  dec convT 1x1->3x3 (GEMM form)                       0.84  0.90  0.033  1.0e-06
  dec 512 res 6x6                                      0.82  0.95  0.043  1.3e-06
  dec convT s2 1024->512                               0.85  0.93  0.045  1.4e-06
  dec convT s2 768->384                                0.82  0.96  0.039  1.2e-06
  dec 384 res 12x12                                    0.84  0.96  0.046  1.4e-06
  dec convT s2 512->256                                0.87  0.98  0.035  1.1e-06
  dec 256 res 24x24                                    0.89  0.98  0.038  1.2e-06
  dec convT s2 320->128                                0.90  0.97  0.030  9.0e-07
  dec 128 res 48x48                                    0.90  0.99  0.031  9.5e-07
  dec convT s2 160->64                                 0.95  0.98  0.023  7.1e-07
  dec 64 res 96x96                                     0.95  0.98  0.023  7.2e-07
  output 80->32 96x96                                  0.90  0.97  0.025  7.6e-07
  sync 7x7 15->32                                      0.89  0.98  0.027  8.4e-07
  sync k5 s(1,2) p1 -> 46x47                           0.89  0.98  0.031  9.5e-07
  sync 64 res 46x47                                    0.94  0.98  0.027  8.1e-07
  sync 64->128 s2 -> 23x24                             0.89  0.97  0.020  6.0e-07
  sync 128 res 23x24                                   0.90  0.98  0.028  8.6e-07
  sync 128->256 s2 -> 12x12                            0.85  0.91  0.027  8.4e-07
  sync 256 res 12x12                                   0.83  0.95  0.037  1.1e-06
  sync 512 s2 6x6 -> 3x3                               0.69  0.91  0.041  1.2e-06
  disc 7x7 3->32 lrelu                                 0.92  0.99  0.043  1.3e-06
  disc k5 s(1,2) p2                                    0.89  0.99  0.026  8.0e-07
  disc k5 64 48x48                                     0.88  0.97  0.037  1.1e-06
  disc k5 s2 64->128                                   0.83  0.96  0.033  1.0e-06
  disc k5 128 24x24                                    0.81  0.97  0.048  1.5e-06
  disc k5 s2 128->256                                  0.73  0.97  0.043  1.3e-06
  disc k5 256 12x12                                    0.75  0.92  0.059  1.8e-06
  disc 3x3 s2 256->512                                 0.79  0.65  0.044  1.3e-06
  disc 512 3x3 6x6                                     0.73  0.95  0.053  1.6e-06
  disc 512 3x3 pad0 -> 1x1                             0.64  0.10  0.048  1.5e-06
  disc 512 1x1                                         0.39  0.07  0.017  5.1e-07
  s3fd conv1_1 3->64 96x128                            0.97  0.95  0.031  9.5e-07
  s3fd conv1_2 64 96x128                               0.91  0.98  0.024  7.4e-07
  s3fd conv2_1 64->128 48x64                           0.90  0.98  0.024  7.2e-07
  s3fd conv2_2 128 48x64                               0.88  0.98  0.035  1.1e-06
  s3fd conv3_1 128->256 24x32                          0.88  0.98  0.030  9.1e-07
  s3fd conv3_2 256 37x52                               0.83  0.97  0.045  1.4e-06
  s3fd conv4_1 256->512 12x16                          0.79  0.95  0.040  1.2e-06
  s3fd conv4_2 512 9x13                                0.83  0.88  0.054  1.6e-06
  s3fd conv5_2 512 3x4                                 0.66  0.91  0.039  1.2e-06
  s3fd fc6 512->1024 k3 p3 3x4                         0.81  0.97  0.478  5.1e-05
  s3fd fc6 512->1024 k3 p3 1x1 -> 5x5                  0.89  0.89  0.478  5.1e-05
  s3fd fc7 1024 1x1 7x8                                0.88  0.97  0.037  1.1e-06
  s3fd conv6_1 1024->256 1x1 7x8                       0.79  0.97  0.036  1.1e-06
  s3fd conv6_2 256->512 s2 7x8                         0.78  0.93  0.032  9.7e-07
  s3fd conv6_2 256->512 s2 5x5 -> 3x3                  0.85  0.94  0.035  1.1e-06
  s3fd conv7_1 512->128 1x1 4x4                        0.84  0.00  0.025  7.6e-07
  s3fd conv7_2 128->256 s2 4x4                         0.72  0.00  0.020  6.0e-07
  s3fd conv7_2 128->256 s2 3x3 -> 2x2                  0.79  0.01  0.017  5.2e-07
  s3fd head plain 256->16 24x32                        0.71  0.95  0.040  1.2e-06
  s3fd head plain 512->16 12x16                        0.72  0.93  0.041  1.2e-06
  s3fd head plain 1024->16 7x8                         0.65  0.26  0.044  1.3e-06
  igemm BN16 BK16 48->48                               0.91  0.98
  igemm BN16 BK32 32->80                               0.89  0.97
  igemm BN16 BK64 64->48                               0.88  0.96
  igemm BN32 BK16 48->96                               0.89  0.98
  igemm BN32 BK32 32->32 s2                            0.82  0.99
  igemm BN32 BK64 64->96                               0.88  0.98
  igemm BN64 BK16 48->192                              0.91  0.98
  igemm BN64 BK32 32->192                              0.94  0.99
  igemm BN64 BK64 64->192                              0.91  0.98
  igemm BN128 BK16 48->128                             0.93  0.99
  igemm BN128 BK32 96->128                             0.91  0.98
  igemm BN128 BK64 64->128                             0.90  0.99
  igemm BN128 res two epilogue passes                  0.92  0.99  0.037  1.1e-06
  igemm ragged bn>1 boxes N=131 3x3                    0.91  0.77
  igemm ragged 13x11 s2                                0.79  0.00
  igemm 37x301 s2 wide rows                            0.93  0.98  0.024  7.4e-07
  mt2 BK64 192 res                                     0.93  0.99  0.039  1.2e-06
  mt2 BK32 32->64 s2                                   0.93  0.99
  mt2 BK64 odd M tiles 1x1 N=67634                     0.96  0.99
  patch BN16 BK16 16 res                               0.91  0.10
  patch BN16 BK32 32->16                               0.84  0.00
  patch BN16 BK64 64->16                               0.78  0.00
  patch BN32 BK16 48->32                               0.87  0.71
  patch BN32 BK64 128->32 two chunks                   0.82  0.96
  patch BN64 BK16 48->64 three chunks                  0.93  0.78
  patch BN64 BK32 32->64                               0.90  0.97
  patch BN16 BK64 128->16 two chunks                   0.76  0.95
  patch ragged 23x24 64 res                            0.89  0.94  0.023  7.0e-07
  fold s1 cin1                                         0.97  0.00
  fold s1 cin3 lrelu                                   0.92  0.99
  fold s1 cin6                                         0.91  0.98
  fold s1 cin15                                        0.89  0.98
  fold s2 cin1                                         0.61  0.00
  fold s2 cin3                                         0.96  0.14
  fold s2 cin6                                         0.94  0.00
  fold s2 cin15                                        0.96  0.99
  convT fused BK32 160->64                             0.95  0.98
  convT fused cin 128 (BK32, four K steps)             0.92  0.99
  convT fused 40x24 in                                 0.92  0.99
  convT phases out_pad 0                               0.92  0.95
  convT 1x1->3x3 GEMM N=1                              0.39  0.90
  convT 1x1->3x3 GEMM N=131                            0.88  0.98  0.049  1.5e-06
  convT s2 cin80 -> 64 (phases, no BK16 fused kernel)  0.93  0.97
"""
import ctypes as C
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import w2l_oracle as O

pytestmark = pytest.mark.gpu

FLAGS = ["W2L_DISABLE_HALO", "W2L_DISABLE_FOLD", "W2L_DISABLE_FOLDS2", "W2L_DISABLE_MT2", "W2L_DISABLE_TMAEPI",
         "W2L_DISABLE_CTFUSED", "W2L_DISABLE_SIDESTREAM", "W2L_DISABLE_PDL"]
F16, BF16, F32X = 0, 1, 2
PREC_NAME = {F16: "f16", BF16: "bf16", F32X: "f32x"}
DTYPE = {F16: torch.float16, BF16: torch.bfloat16}
MANT = {F16: 10, BF16: 7}
MIN_SUB = {F16: 2.0 ** -24, BF16: 2.0 ** -133}
ACC = 2.0 ** -16      # fp32 accumulation term of the 16-bit bars
ACC_X2 = 2.0 ** -15   # the F32X bar
ALL_OFF = tuple(FLAGS)

# ------------------------------------------------------------------------------------------------------------------
# contexts: one per (precision, switch set), created with the switches in the environment, closed at module teardown
# ------------------------------------------------------------------------------------------------------------------
_CTX = {}


def _ctx(prec, off=()):
    from wav2lip_b200 import _lib
    key = (prec, tuple(sorted(off)))
    if key not in _CTX:
        old = {k: os.environ.get(k) for k in FLAGS}
        try:
            for k in FLAGS:
                os.environ.pop(k, None)
            for k in off:
                os.environ[k] = "1"
            _CTX[key] = _lib.Context(0, prec)   # the W2L_DISABLE_* switches are read here
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    return _CTX[key]


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in _CTX.values():
        c.close()
    _CTX.clear()


# ------------------------------------------------------------------------------------------------------------------
# reference arithmetic
# ------------------------------------------------------------------------------------------------------------------
def round16(t, prec):
    return t if prec == F32X else t.to(DTYPE[prec]).double()


def ulp16(a, prec):
    """Spacing of the 16-bit type at |a| (float64 in, float64 out): 2^(e-1-mant) for |a| in [2^(e-1), 2^e)."""
    a = a.abs()
    _m, e = torch.frexp(a)
    u = torch.ldexp(torch.ones_like(a), e - 1 - MANT[prec])
    return torch.where(a == 0, torch.full_like(a, MIN_SUB[prec]), torch.clamp(u, min=MIN_SUB[prec]))


def lo_step(a):
    """F32X stores y as hi + lo in two fp16 planes, lo = fp16(y - hi): the lo rounding is at most half an fp16 step of a
    value at most half an fp16 step of y.  About 2^-22 |y|; it matters only where fp16 makes lo subnormal (|y| < ~2^-3),
    and there only when mag is tiny too (an output that is a bias alone, like fc6's padding-only border)."""
    return 0.5 * ulp16(0.5 * ulp16(a, F16), F16)


def _row_geom(row):
    kind, cin, cout, k, s, p, op, res = row
    return kind, cin, cout, O._pair(k), O._pair(s), O._pair(p), op, res


def fold_bn(sd, prefix, kind):
    """(scale, shift) float64 from the fp32 parameters, as fold_bn_kernel folds them."""
    b = sd[f"{prefix}.conv_block.0.bias"].double()
    if kind in ("n", "r", "p"):   # no BatchNorm: scale 1, shift = conv bias
        return torch.ones_like(b), b
    g = sd[f"{prefix}.conv_block.1.weight"].double()
    be = sd[f"{prefix}.conv_block.1.bias"].double()
    m = sd[f"{prefix}.conv_block.1.running_mean"].double()
    v = sd[f"{prefix}.conv_block.1.running_var"].double()
    s = g / torch.sqrt(v + O.BN_EPS)
    return s, (b - m) * s + be


def reference(x, sd, prefix, row, prec, round_out=True):
    """float64 (ref, mag) of one block on the input x the kernel saw (x already carries the kernel's operand rounding
    for an exported activation; a caller tensor is rounded here)."""
    kind, _cin, _cout, k, s, p, op, res = _row_geom(row)
    dev = "cuda"
    xr = round16(x.to(dev, torch.float64), prec)
    w = round16(sd[f"{prefix}.conv_block.0.weight"].to(dev, torch.float64), prec)
    if kind == "t":
        conv = lambda a, b: F.conv_transpose2d(a, b, stride=s, padding=p, output_padding=op)
    else:
        conv = lambda a, b: F.conv2d(a, b, stride=s, padding=p)
    z = conv(xr, w)
    za = conv(xr.abs(), w.abs())
    scale, shift = (t.to(dev).view(1, -1, 1, 1) for t in fold_bn(sd, prefix, kind))
    v = scale * z + shift
    mag = scale.abs() * za + shift.abs()
    if res:
        v = v + xr
        mag = mag + xr.abs()
    if kind == "n":
        v = F.leaky_relu(v, 0.01)
    elif kind != "p":
        v = F.relu(v)
    if prec != F32X and round_out:
        v = round16(v, prec)
    return v, mag


def compare(y, ref, mag, prec, what=""):
    """Asserts the bars of the module docstring; returns (max err/bar, max err/mag, bias)."""
    y = y.to(ref.device, torch.float64)
    assert y.shape == ref.shape, (what, tuple(y.shape), tuple(ref.shape))
    assert torch.isfinite(y).all(), f"{what}: non-finite output"
    err = (y - ref).abs()
    if prec == F32X:
        bar = ACC_X2 * mag + lo_step(torch.maximum(y.abs(), ref.abs()))
    else:
        bar = ulp16(torch.maximum(y.abs(), ref.abs()), prec) + ACC * mag
    ratio = (err / bar).max().item()
    emag = (err / mag.clamp(min=1e-300)).max().item()
    bias = 0.0
    if prec != F32X and ref.numel() >= 10_000:
        sel = ref.abs() > ACC * mag
        bias = (torch.sign(ref[sel]) * (y[sel] - ref[sel]) / ulp16(ref[sel], prec)).mean().item()
    if ratio > 1.0:
        i = int(torch.argmax(err / bar))
        idx = tuple(int(t) for t in torch.unravel_index(torch.tensor(i), ref.shape))
        raise AssertionError(f"{what} [{PREC_NAME[prec]}]: max err/bar {ratio:.3g} at {idx}: y {y.flatten()[i].item():.9g} "
                             f"ref {ref.flatten()[i].item():.9g} mag {mag.flatten()[i].item():.4g}")
    assert abs(bias) <= 0.05, f"{what} [{PREC_NAME[prec]}]: rounding bias {bias:.4f} ulp (round-to-nearest gives ~0)"
    return ratio, emag, bias


# ------------------------------------------------------------------------------------------------------------------
# one block through w2l_conv_block_forward on a private context
# ------------------------------------------------------------------------------------------------------------------
KIND = {"c": 0, "t": 1, "n": 2, "p": 3, "r": 4}   # W2L_BLOCK_*


def block_forward(ctx, row, x, sd, prefix="b"):
    from wav2lip_b200 import _lib
    kind, cin, cout, (kh, kw), (sh, sw), (ph, pw), op, res = _row_geom(row)
    li = _lib.LayerInfo()
    li.name = b"b"
    li.kind = KIND[kind]
    li.cin, li.cout, li.kh, li.kw, li.sh, li.sw, li.ph, li.pw = cin, cout, kh, kw, sh, sw, ph, pw
    li.out_pad = op
    li.residual = 1 if res else 0
    n, _, h, w = x.shape
    if kind == "t":
        ho, wo = (h - 1) * sh - 2 * ph + kh + op, (w - 1) * sw - 2 * pw + kw + op
    else:
        ho, wo = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    dev = lambda t: t.detach().to("cuda", torch.float32).contiguous() if t is not None else None
    xd = dev(x)
    t = {k: dev(sd.get(f"{prefix}.conv_block.{k}")) for k in ("0.weight", "0.bias", "1.weight", "1.bias", "1.running_mean",
                                                                "1.running_var")}
    y = torch.empty((n, cout, ho, wo), device="cuda", dtype=torch.float32)
    ptr = lambda a: C.c_void_p(a.data_ptr()) if a is not None else C.c_void_p(0)
    torch.cuda.synchronize()
    _lib.check(ctx.lib.w2l_conv_block_forward(ctx.h, C.byref(li), ptr(xd), n, h, w, ptr(t["0.weight"]), ptr(t["0.bias"]),
                                              ptr(t["1.weight"]), ptr(t["1.bias"]), ptr(t["1.running_mean"]),
                                              ptr(t["1.running_var"]), ptr(y), C.c_void_p(0)))
    return y


def _tensors(row, seed, N, H, W):
    g = torch.Generator().manual_seed(seed)
    # _block_tensors adds BatchNorm tensors for every kind but "n"; the plain and ReLU kinds have none
    sd = O._block_tensors("b", ("n",) + tuple(row[1:]) if row[0] in ("r", "p") else row, g, 1.0)
    x = torch.rand((N, row[1], H, W), generator=g) * 2 - 0.5
    return sd, x


# ------------------------------------------------------------------------------------------------------------------
# cases.  expect: "<family><BN>.<BK>[m2][e][f]" for every launch of the case (I = generic, P = patch, T = fused
# transposed conv; m2 = two M tiles per CTA, e = staged TMA epilogue, f = K-folded), "*" = not asserted
# ------------------------------------------------------------------------------------------------------------------
def _c(cin, cout, k, s, p, res=False):
    return ("c", cin, cout, k, s, p, 0, res)


def _t(cin, cout, k, s, p, op=0):
    return ("t", cin, cout, k, s, p, op, False)


def _n(cin, cout, k, s, p):
    return ("n", cin, cout, k, s, p, 0, False)


def _r(cin, cout, k, s, p):
    return ("r", cin, cout, k, s, p, 0, False)


def _p(cin, cout, k, s, p):
    return ("p", cin, cout, k, s, p, 0, False)


# every distinct block geometry of the generator, SyncNet and the disc (input N, H, W), default-dispatch kernel in F16
GEOMS = [
    ("gen 7x7 6->16 96x96", _c(6, 16, 7, 1, 3), 2, 96, 96, "P16.64f"),
    ("gen 16->32 s2 96x96", _c(16, 32, 3, 2, 1), 2, 96, 96, "I32.64ef"),
    ("gen 32 res 48x48", _c(32, 32, 3, 1, 1, True), 2, 48, 48, "P32.32"),
    ("gen 32->64 s2 48x48", _c(32, 64, 3, 2, 1), 2, 48, 48, "I32.32e"),
    ("gen 64 res 24x24", _c(64, 64, 3, 1, 1, True), 2, 24, 24, "P64.64"),
    ("gen 64->128 s2 24x24", _c(64, 128, 3, 2, 1), 2, 24, 24, "I32.64e"),
    ("gen 128 res 12x12", _c(128, 128, 3, 1, 1, True), 3, 12, 12, "I32.64e"),
    ("gen 128->256 s2 12x12", _c(128, 256, 3, 2, 1), 3, 12, 12, "I32.64e"),
    ("gen 256 res 6x6", _c(256, 256, 3, 1, 1, True), 3, 6, 6, "I32.64e"),
    ("gen 256->512 s2 6x6", _c(256, 512, 3, 2, 1), 3, 6, 6, "I32.64e"),
    ("gen 512 res 3x3", _c(512, 512, 3, 1, 1, True), 3, 3, 3, "I32.64e"),
    ("gen 512 3x3 pad0 -> 1x1", _c(512, 512, 3, 1, 0), 3, 3, 3, "I32.64e"),
    ("gen 512 1x1", _c(512, 512, 1, 1, 0), 5, 1, 1, "I32.64e"),
    ("audio 1->32 80x16", _c(1, 32, 3, 1, 1), 2, 80, 16, "P32.32f"),
    ("audio 32 res 80x16", _c(32, 32, 3, 1, 1, True), 2, 80, 16, "P32.32"),
    ("audio 32->64 s(3,1)", _c(32, 64, 3, (3, 1), 1), 2, 80, 16, "I32.32e"),
    ("audio 64 res 27x16", _c(64, 64, 3, 1, 1, True), 2, 27, 16, "P64.64"),
    ("audio 64->128 s3", _c(64, 128, 3, 3, 1), 2, 27, 16, "I32.64e"),
    ("audio 128 res 9x6", _c(128, 128, 3, 1, 1, True), 2, 9, 6, "I32.64e"),
    ("audio 128->256 s(3,2)", _c(128, 256, 3, (3, 2), 1), 2, 9, 6, "I32.64e"),
    ("audio 256 res 3x3", _c(256, 256, 3, 1, 1, True), 2, 3, 3, "I32.64e"),
    ("audio 256->512 3x3 pad0", _c(256, 512, 3, 1, 0), 2, 3, 3, "I32.64e"),
    ("dec convT 1x1->3x3 (GEMM form)", _t(1024, 512, 3, 1, 0), 3, 1, 1, "I32.64e"),
    ("dec 512 res 6x6", _c(512, 512, 3, 1, 1, True), 2, 6, 6, "I32.64e"),
    ("dec convT s2 1024->512", _t(1024, 512, 3, 2, 1, 1), 2, 3, 3, "I32.64e"),
    ("dec convT s2 768->384", _t(768, 384, 3, 2, 1, 1), 1, 6, 6, "I32.64e"),
    ("dec 384 res 12x12", _c(384, 384, 3, 1, 1, True), 1, 12, 12, "I32.64e"),
    ("dec convT s2 512->256", _t(512, 256, 3, 2, 1, 1), 1, 12, 12, "I32.64e"),
    ("dec 256 res 24x24", _c(256, 256, 3, 1, 1, True), 1, 24, 24, "I32.64e"),
    ("dec convT s2 320->128", _t(320, 128, 3, 2, 1, 1), 1, 24, 24, "I32.64e"),
    ("dec 128 res 48x48", _c(128, 128, 3, 1, 1, True), 1, 48, 48, "I32.64e"),
    ("dec convT s2 160->64", _t(160, 64, 3, 2, 1, 1), 1, 48, 48, "T64.32"),
    ("dec 64 res 96x96", _c(64, 64, 3, 1, 1, True), 1, 96, 96, "P64.64"),
    ("output 80->32 96x96", _c(80, 32, 3, 1, 1), 1, 96, 96, "P32.16"),
    ("sync 7x7 15->32", _c(15, 32, 7, 1, 3), 2, 48, 96, "P32.64f"),
    ("sync k5 s(1,2) p1 -> 46x47", _c(32, 64, 5, (1, 2), 1), 2, 48, 96, "I32.32e"),
    ("sync 64 res 46x47", _c(64, 64, 3, 1, 1, True), 2, 46, 47, "P64.64"),
    ("sync 64->128 s2 -> 23x24", _c(64, 128, 3, 2, 1), 2, 46, 47, "I32.64e"),
    ("sync 128 res 23x24", _c(128, 128, 3, 1, 1, True), 2, 23, 24, "I32.64e"),
    ("sync 128->256 s2 -> 12x12", _c(128, 256, 3, 2, 1), 2, 23, 24, "I32.64e"),
    ("sync 256 res 12x12", _c(256, 256, 3, 1, 1, True), 2, 12, 12, "I32.64e"),
    ("sync 512 s2 6x6 -> 3x3", _c(512, 512, 3, 2, 1), 2, 6, 6, "I32.64e"),
    ("disc 7x7 3->32 lrelu", _n(3, 32, 7, 1, 3), 2, 48, 96, "P32.64f"),
    ("disc k5 s(1,2) p2", _n(32, 64, 5, (1, 2), 2), 2, 48, 96, "I32.32e"),
    ("disc k5 64 48x48", _n(64, 64, 5, 1, 2), 2, 48, 48, "I32.64e"),
    ("disc k5 s2 64->128", _n(64, 128, 5, 2, 2), 2, 48, 48, "I32.64e"),
    ("disc k5 128 24x24", _n(128, 128, 5, 1, 2), 2, 24, 24, "I32.64e"),
    ("disc k5 s2 128->256", _n(128, 256, 5, 2, 2), 2, 24, 24, "I32.64e"),
    ("disc k5 256 12x12", _n(256, 256, 5, 1, 2), 1, 12, 12, "I32.64e"),
    ("disc 3x3 s2 256->512", _n(256, 512, 3, 2, 1), 2, 12, 12, "I32.64e"),
    ("disc 512 3x3 6x6", _n(512, 512, 3, 1, 1), 2, 6, 6, "I32.64e"),
    ("disc 512 3x3 pad0 -> 1x1", _n(512, 512, 3, 1, 0), 2, 3, 3, "I32.64e"),
    ("disc 512 1x1", _n(512, 512, 1, 1, 0), 2, 1, 1, "I32.64e"),
]

# every distinct S3FD layer geometry (conv + ReLU backbone, plain 16-channel heads) at sizes its plans produce: the
# backbone of a 96x128 frame, the odd maps of 150x210, fc6 (k3 pad 3) on the 1x1 pool5 of a 32x32 frame, the stride-2
# convs down to 3x3 and 2x2 inputs
S3FD_GEOMS = [
    ("s3fd conv1_1 3->64 96x128", _r(3, 64, 3, 1, 1), 2, 96, 128, "P64.32f"),
    ("s3fd conv1_2 64 96x128", _r(64, 64, 3, 1, 1), 2, 96, 128, "P64.64"),
    ("s3fd conv2_1 64->128 48x64", _r(64, 128, 3, 1, 1), 2, 48, 64, "I32.64e"),
    ("s3fd conv2_2 128 48x64", _r(128, 128, 3, 1, 1), 2, 48, 64, "I32.64e"),
    ("s3fd conv3_1 128->256 24x32", _r(128, 256, 3, 1, 1), 2, 24, 32, "I32.64e"),
    ("s3fd conv3_2 256 37x52", _r(256, 256, 3, 1, 1), 1, 37, 52, "I32.64e"),
    ("s3fd conv4_1 256->512 12x16", _r(256, 512, 3, 1, 1), 2, 12, 16, "I32.64e"),
    ("s3fd conv4_2 512 9x13", _r(512, 512, 3, 1, 1), 1, 9, 13, "I32.64e"),
    ("s3fd conv5_2 512 3x4", _r(512, 512, 3, 1, 1), 2, 3, 4, "I32.64e"),
    ("s3fd fc6 512->1024 k3 p3 3x4", _r(512, 1024, 3, 1, 3), 2, 3, 4, "I32.64e"),
    ("s3fd fc6 512->1024 k3 p3 1x1 -> 5x5", _r(512, 1024, 3, 1, 3), 3, 1, 1, "I32.64e"),
    ("s3fd fc7 1024 1x1 7x8", _r(1024, 1024, 1, 1, 0), 2, 7, 8, "I32.64e"),
    ("s3fd conv6_1 1024->256 1x1 7x8", _r(1024, 256, 1, 1, 0), 2, 7, 8, "I32.64e"),
    ("s3fd conv6_2 256->512 s2 7x8", _r(256, 512, 3, 2, 1), 2, 7, 8, "I32.64e"),
    ("s3fd conv6_2 256->512 s2 5x5 -> 3x3", _r(256, 512, 3, 2, 1), 3, 5, 5, "I32.64e"),
    ("s3fd conv7_1 512->128 1x1 4x4", _r(512, 128, 1, 1, 0), 2, 4, 4, "I32.64e"),
    ("s3fd conv7_2 128->256 s2 4x4", _r(128, 256, 3, 2, 1), 2, 4, 4, "I32.64e"),
    ("s3fd conv7_2 128->256 s2 3x3 -> 2x2", _r(128, 256, 3, 2, 1), 3, 3, 3, "I32.64e"),
    ("s3fd head plain 256->16 24x32", _p(256, 16, 3, 1, 1), 2, 24, 32, "I16.64e"),
    ("s3fd head plain 512->16 12x16", _p(512, 16, 3, 1, 1), 2, 12, 16, "I16.64e"),
    ("s3fd head plain 1024->16 7x8", _p(1024, 16, 3, 1, 1), 2, 7, 8, "I16.64e"),
]

# cases aimed at the dispatch boundaries (default dispatch, F16 and BF16)
DISPATCH = [
    # generic kernel: every BN x BK instantiation
    ("igemm BN16 BK16 48->48", _c(48, 48, 3, 1, 1), 3, 24, 24, "I16.16e"),
    ("igemm BN16 BK32 32->80", _c(32, 80, 3, 1, 1), 3, 20, 20, "I16.32e"),
    ("igemm BN16 BK64 64->48", _c(64, 48, 3, 1, 1), 3, 24, 24, "I16.64e"),
    ("igemm BN32 BK16 48->96", _c(48, 96, 3, 1, 1), 3, 24, 24, "I32.16e"),
    ("igemm BN32 BK32 32->32 s2", _c(32, 32, 3, 2, 1), 2, 48, 48, "I32.32e"),
    ("igemm BN32 BK64 64->96", _c(64, 96, 3, 1, 1), 3, 24, 24, "I32.64e"),
    ("igemm BN64 BK16 48->192", _c(48, 192, 3, 1, 1), 10, 24, 24, "I64.16e"),
    ("igemm BN64 BK32 32->192", _c(32, 192, 3, 1, 1), 10, 24, 24, "I64.32e"),
    ("igemm BN64 BK64 64->192", _c(64, 192, 3, 1, 1), 10, 24, 24, "I64.64e"),
    ("igemm BN128 BK16 48->128", _c(48, 128, 3, 1, 1), 8, 48, 48, "I128.16e"),
    ("igemm BN128 BK32 96->128", _c(96, 128, 3, 1, 1), 8, 48, 48, "I128.32e"),
    ("igemm BN128 BK64 64->128", _c(64, 128, 3, 1, 1), 8, 48, 48, "I128.64e"),
    ("igemm BN128 res two epilogue passes", _c(128, 128, 3, 1, 1, True), 30, 24, 24, "I128.64e"),
    ("igemm ragged bn>1 boxes N=131 3x3", _c(64, 64, 3, 1, 1, True), 131, 3, 3, "I32.64e"),
    ("igemm ragged 13x11 s2", _c(32, 64, 3, 2, 1), 5, 13, 11, "I32.32e"),
    ("igemm 37x301 s2 wide rows", _c(32, 64, 3, 2, 1), 1, 73, 601, "I32.32e"),
    # two M tiles per CTA
    ("mt2 BK64 192 res", _c(192, 192, 3, 1, 1, True), 39, 24, 24, "I64.64m2e"),
    ("mt2 BK32 32->64 s2", _c(32, 64, 3, 2, 1), 30, 96, 96, "I64.32m2e"),
    ("mt2 BK64 odd M tiles 1x1 N=67634", _c(64, 64, 1, 1, 0), 67634, 1, 1, "I64.64m2e"),
    # patch kernel
    ("patch BN16 BK16 16 res", _c(16, 16, 3, 1, 1, True), 2, 48, 48, "P16.16"),
    ("patch BN16 BK32 32->16", _c(32, 16, 3, 1, 1), 2, 24, 24, "P16.32"),
    ("patch BN16 BK64 64->16", _c(64, 16, 3, 1, 1), 2, 24, 24, "P16.64"),
    ("patch BN32 BK16 48->32", _c(48, 32, 3, 1, 1), 2, 24, 24, "P32.16"),
    ("patch BN32 BK64 128->32 two chunks", _c(128, 32, 3, 1, 1), 2, 24, 24, "P32.64"),
    ("patch BN64 BK16 48->64 three chunks", _c(48, 64, 3, 1, 1), 2, 24, 24, "P64.16"),
    ("patch BN64 BK32 32->64", _c(32, 64, 3, 1, 1), 2, 24, 24, "P64.32"),
    ("patch BN16 BK64 128->16 two chunks", _c(128, 16, 3, 1, 1), 2, 24, 24, "P16.64"),
    ("patch ragged 23x24 64 res", _c(64, 64, 3, 1, 1, True), 3, 23, 24, "P64.64"),
    # K-folded first layers
    ("fold s1 cin1", _c(1, 32, 3, 1, 1), 3, 80, 16, "P32.32f"),
    ("fold s1 cin3 lrelu", _n(3, 32, 7, 1, 3), 2, 48, 96, "P32.64f"),
    ("fold s1 cin6", _c(6, 16, 7, 1, 3), 2, 96, 96, "P16.64f"),
    ("fold s1 cin15", _c(15, 32, 7, 1, 3), 2, 48, 96, "P32.64f"),
    ("fold s2 cin1", _c(1, 32, 3, 2, 1), 3, 80, 16, "I32.32ef"),
    ("fold s2 cin3", _c(3, 32, 3, 2, 1), 2, 96, 96, "I32.32ef"),
    ("fold s2 cin6", _c(6, 32, 3, 2, 1), 2, 96, 96, "I32.32ef"),
    ("fold s2 cin15", _c(15, 32, 3, 2, 1), 2, 96, 96, "I32.64ef"),
    # transposed convs
    ("convT fused BK32 160->64", _t(160, 64, 3, 2, 1, 1), 2, 48, 48, "T64.32"),
    ("convT fused cin 128 (BK32, four K steps)", _t(128, 64, 3, 2, 1, 1), 2, 24, 24, "T64.32"),
    ("convT fused 40x24 in", _t(128, 64, 3, 2, 1, 1), 2, 40, 24, "T64.32"),
    ("convT phases out_pad 0", _t(128, 64, 3, 2, 1, 0), 2, 12, 12, "I32.64e"),
    ("convT 1x1->3x3 GEMM N=1", _t(1024, 512, 3, 1, 0), 1, 1, 1, "I32.64e"),
    ("convT 1x1->3x3 GEMM N=131", _t(1024, 512, 3, 1, 0), 131, 1, 1, "I64.64e"),
    ("convT s2 cin80 -> 64 (phases, no BK16 fused kernel)", _t(80, 64, 3, 2, 1, 1), 2, 24, 24, "P64.16"),
]

def _short(k):
    return ("IPT"[k["family"]] + f"{k['bn']}.{k['bk']}" + ("m2" if k["mt"] == 2 else "") + ("e" if k["tma_epi"] else "")
            + ("f" if k["fold"] else ""))


def _check_kernels(ks, expect, prec, off, what):
    assert ks, f"{what}: no conv launch reported"
    for k in ks:
        assert k["bf16"] == (1 if prec == BF16 else 0) and k["x2"] == (1 if prec == F32X else 0) and not k["head"], (what, k)
    got = [_short(k) for k in ks]
    if prec == F32X or set(off) == set(ALL_OFF):
        # the specialised paths are off: generic kernel, direct epilogue, plain K (F32X keeps two M tiles per CTA)
        assert all(k["family"] == 0 and not k["tma_epi"] and not k["fold"] for k in ks), (what, got)
        assert prec == F32X or all(k["mt"] == 1 for k in ks), (what, got)
        return
    if expect == "*" or off:
        return
    assert all(g == expect for g in got), f"{what}: expected {expect} for every launch, dispatch chose {got}"


# results of passing cases, shared by the coverage test: (case id, precision, off) -> list of kernel rows
_SEEN = {}
_REFS = {}


def run_case(case, prec, off=(), repeat=True):
    name, row, N, H, W, expect = case
    key = (name, prec, tuple(sorted(off)))
    if key in _SEEN:
        return _SEEN[key]
    sd, x = _tensors(row, 1234, N, H, W)
    ctx = _ctx(prec, off)
    rk = (name, prec)
    if rk not in _REFS:
        if len(_REFS) >= 4:
            _REFS.clear()   # a few references at a time (they can be large)
        _REFS[rk] = reference(x, sd, "b", row, prec)
    ref, mag = _REFS[rk]
    if prec == F16:
        ctx.f16_overflow(clear=True)
    y = block_forward(ctx, row, x, sd)
    ks = ctx.plan_kernels(-1)
    if prec == F16:
        assert not ctx.f16_overflow(clear=True), f"{name}: fp16 range flag set by an in-range case"
    _check_kernels(ks, expect, prec, off, name)
    if repeat:
        y2 = block_forward(ctx, row, x, sd)
        assert torch.equal(y, y2), f"{name} [{PREC_NAME[prec]}]: two runs differ"
    stats = compare(y, ref, mag, prec, name)
    _SEEN[key] = {"kernels": ks, "stats": stats}
    return _SEEN[key]


GEOM_MODES = [(F16, ()), (F16, ALL_OFF), (BF16, ()), (BF16, ALL_OFF), (F32X, ())]
GEOM_MODE_IDS = ["f16", "f16-generic", "bf16", "bf16-generic", "f32x"]


@pytest.mark.parametrize("mode", GEOM_MODES, ids=GEOM_MODE_IDS)
@pytest.mark.parametrize("case", GEOMS, ids=[c[0] for c in GEOMS])
def test_block_geometry_matches_float64(case, mode):
    prec, off = mode
    run_case(case, prec, off)


@pytest.mark.parametrize("mode", GEOM_MODES, ids=GEOM_MODE_IDS)
@pytest.mark.parametrize("case", S3FD_GEOMS, ids=[c[0] for c in S3FD_GEOMS])
def test_s3fd_geometry_matches_float64(case, mode):
    prec, off = mode
    run_case(case, prec, off)


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", DISPATCH, ids=[c[0] for c in DISPATCH])
def test_dispatch_boundary_matches_float64(case, prec):
    run_case(case, prec)


F32X_CASES = [c for c in DISPATCH if c[0] in ("convT 1x1->3x3 GEMM N=131", "igemm BN128 res two epilogue passes",
                                               "patch ragged 23x24 64 res", "igemm 37x301 s2 wide rows", "mt2 BK64 192 res")]


@pytest.mark.parametrize("case", F32X_CASES, ids=[c[0] for c in F32X_CASES])
def test_dispatch_geometry_f32x(case):
    """The 1x1 -> 3x3 transposed conv takes the phase path in F32X; the others check the split residual planes."""
    r = run_case(case, F32X)
    if case[1][0] == "t":
        assert len(r["kernels"]) == 1 and r["kernels"][0]["family"] == 0


def test_fused_convt_falls_back_for_cin_not_multiple_of_32():
    """k3 s2 p1 op1 transposed convs with 64 output channels and cin 80 have no fused kernel (it steps K by 32
    channels): four phase launches, each on the patch kernel."""
    case = [c for c in DISPATCH if c[0].startswith("convT s2 cin80")][0]
    for prec in (F16, BF16):
        ks = run_case(case, prec)["kernels"]
        assert len(ks) == 4 and all(k["family"] != 2 for k in ks), [_short(k) for k in ks]


def test_phase_path_out_pad0_has_unequal_phases():
    case = [c for c in DISPATCH if c[0] == "convT phases out_pad 0"][0]
    ks = run_case(case, F16)["kernels"]
    assert len(ks) == 4 and all(k["family"] == 0 for k in ks), [_short(k) for k in ks]


def test_mt2_odd_m_tiles():
    case = [c for c in DISPATCH if c[0].startswith("mt2 BK64 odd M tiles")][0]
    ks = run_case(case, F16)["kernels"]
    assert ks[0]["mt"] == 2 and ks[0]["m_tiles"] % 2 == 1, ks


# ------------------------------------------------------------------------------------------------------------------
# switches that keep the K order of every output: bit-identical results
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flag,case_name", [
    ("W2L_DISABLE_MT2", "mt2 BK64 192 res"), ("W2L_DISABLE_MT2", "mt2 BK32 32->64 s2"),
    ("W2L_DISABLE_TMAEPI", "igemm BN128 res two epilogue passes"), ("W2L_DISABLE_TMAEPI", "igemm ragged bn>1 boxes N=131 3x3"),
    ("W2L_DISABLE_PDL", "patch ragged 23x24 64 res"), ("W2L_DISABLE_PDL", "convT fused BK32 160->64"),
])
@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_switch_is_bit_identical(flag, case_name, prec):
    case = [c for c in DISPATCH if c[0] == case_name][0]
    _name, row, N, H, W, _e = case
    sd, x = _tensors(row, 1234, N, H, W)
    y_on = block_forward(_ctx(prec), row, x, sd)
    k_on = _ctx(prec).plan_kernels(-1)
    y_off = block_forward(_ctx(prec, (flag,)), row, x, sd)
    k_off = _ctx(prec, (flag,)).plan_kernels(-1)
    if flag == "W2L_DISABLE_MT2":
        assert k_on[0]["mt"] == 2 and k_off[0]["mt"] == 1
    if flag == "W2L_DISABLE_TMAEPI":
        assert k_on[0]["tma_epi"] == 1 and k_off[0]["tma_epi"] == 0
    assert torch.equal(y_on, y_off), f"{flag}: max diff {(y_on - y_off).abs().max().item():.3g}"


# ------------------------------------------------------------------------------------------------------------------
# coverage: every compiled instantiation the block entry can reach met the float64 reference in fp16 and bf16
# ------------------------------------------------------------------------------------------------------------------
def test_every_reachable_instantiation_is_covered():
    from wav2lip_b200 import _lib
    table = [k for k in _lib.kernel_table() if not k["head"]]   # the heads are covered by the network checks
    assert len(table) == 2 * (12 + 2 + 9 + 1)
    seen = set()
    for prec in (F16, BF16):
        for case in GEOMS + S3FD_GEOMS + DISPATCH:
            for k in run_case(case, prec)["kernels"]:
                seen.add((k["family"], k["bn"], k["bk"], k["mt"], k["bf16"]))
    missing = [(k["family"], k["bn"], k["bk"], k["mt"], k["bf16"]) for k in table
               if (k["family"], k["bn"], k["bk"], k["mt"], k["bf16"]) not in seen]
    assert not missing, f"compiled conv instantiations no parity case reaches (family, BN, BK, MT, bf16): {missing}"


# ------------------------------------------------------------------------------------------------------------------
# fp16 range flag, per kernel family: exactly one output element beyond 65504 sets it, the in-range neighbour does not
# ------------------------------------------------------------------------------------------------------------------
def _overflow_tensors(row, N, H, W, big):
    kind, cin, cout = row[0], row[1], row[2]
    sd, x = _tensors(row, 99, N, H, W)
    x = x * 0.1
    w = sd["b.conv_block.0.weight"] * 0.1
    kh, kw = O._pair(row[3])
    if kind == "t":
        w[0, :] = 0.0
        w[0, 0, kh // 2, kw // 2] = 2.0
    else:
        w[:, 0] = 0.0
        w[0, 0, kh // 2, kw // 2] = 2.0
    sd["b.conv_block.0.weight"] = w
    sd["b.conv_block.1.weight"] = torch.ones(cout)
    sd["b.conv_block.1.bias"] = torch.zeros(cout)
    sd["b.conv_block.1.running_mean"] = torch.zeros(cout)
    sd["b.conv_block.1.running_var"] = torch.ones(cout) - O.BN_EPS
    x[:, 0] = 0.0
    x[N - 1, 0, H // 2, W // 2] = big     # one input element -> one output element of channel 0
    return sd, x


@pytest.mark.parametrize("family,row,N,H,W,off,expect", [
    ("generic direct epilogue", _c(64, 128, 3, 2, 1), 2, 24, 24, ("W2L_DISABLE_TMAEPI",), "I32.64"),
    ("generic staged epilogue", _c(64, 128, 3, 2, 1), 2, 24, 24, (), "I32.64e"),
    ("patch", _c(64, 64, 3, 1, 1, True), 2, 23, 24, (), "P64.64"),
    ("fused convT", _t(128, 64, 3, 2, 1, 1), 2, 24, 24, (), "T64.32"),
], ids=["generic-direct", "generic-staged", "patch", "fused-convT"])
def test_f16_range_flag_per_family(family, row, N, H, W, off, expect):
    ctx = _ctx(F16, off)
    for big, flagged in ((40000.0, True), (10000.0, False)):
        sd, x = _overflow_tensors(row, N, H, W, big)
        ctx.f16_overflow(clear=True)
        y = block_forward(ctx, row, x, sd)
        assert _short(ctx.plan_kernels(-1)[0]) == expect, ctx.plan_kernels(-1)
        assert ctx.f16_overflow(clear=True) == flagged, (family, big)
        assert int(torch.isinf(y).sum()) == (1 if flagged else 0)


# ------------------------------------------------------------------------------------------------------------------
# networks, one layer at a time: the reference is fed the GPU's own export of each block's input
# ------------------------------------------------------------------------------------------------------------------
NET_SWITCHES = [()] + [(f,) for f in FLAGS] + [ALL_OFF]
NET_SWITCH_IDS = ["all-on"] + [f.replace("W2L_DISABLE_", "no-").lower() for f in FLAGS] + ["generic-only"]
_NET_OUT = {}


def _load(ctx, net, sd):
    dev ={k: v.to("cuda", torch.float32).contiguous() for k, v in sd.items() if v.dtype != torch.long}
    ctx.load_weights(net, {k: (v.data_ptr(), v.numel()) for k, v in dev.items()})
    torch.cuda.synchronize()
    return dev


def _export(ctx, net, i):
    from wav2lip_b200 import _lib
    n, c, h, w = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    r = ctx.lib.w2l_debug_layer_output(ctx.h, net, i, None, C.byref(n), C.byref(c), C.byref(h), C.byref(w), None)
    if r != 0:
        return None
    y = torch.empty((n.value, c.value, h.value, w.value), device="cuda", dtype=torch.float32)
    _lib.check(ctx.lib.w2l_debug_layer_output(ctx.h, net, i, C.c_void_p(y.data_ptr()), None, None, None, None, None))
    torch.cuda.synchronize()
    return y


def _check_chain(ctx, net, layers, sd, inputs, prec, items, what):
    """layers: [(name, row)] in table order; inputs: name -> float32 block input (or a callable of the exports)."""
    outs, worst = {}, 0.0
    for i, (name, row) in enumerate(layers):
        y = _export(ctx, net, i)
        outs[name] = y
        x = inputs(name, outs)
        if y is None or x is None:
            continue
        ref, mag = reference(x[items], sd, name, row, prec)
        worst = max(worst, compare(y[items], ref, mag, prec, f"{what} {name}")[0])
    return outs, worst


def _generator_inputs(mel, face, prec):
    layers = O.generator_layers()
    names = [n for n, _ in layers]
    enc_last = {i: f"face_encoder_blocks.{i}.{len(b) - 1}" for i, b in enumerate(O.GEN_FACE_ENCODER)}
    dec_last = {i: f"face_decoder_blocks.{i}.{len(b) - 1}" for i, b in enumerate(O.GEN_FACE_DECODER)}

    def inputs(name, outs):
        k = names.index(name)
        if name == "face_encoder_blocks.0.0":
            return face.cuda()
        if name == "audio_encoder.0":
            return mel.cuda()
        if name == "face_decoder_blocks.0.0":
            return outs["audio_encoder.12"]
        if name == "output_block.0":
            a, b = outs.get(dec_last[6]), outs.get(enc_last[0])
            return None if a is None or b is None else torch.cat([a, b], 1)
        if name.startswith("face_decoder_blocks.") and name.endswith(".0"):
            s = int(name.split(".")[1])
            a, b = outs.get(dec_last[s - 1]), outs.get(enc_last[6 - (s - 1)])
            return None if a is None or b is None else torch.cat([a, b], 1)
        if name.startswith("face_encoder_blocks.") and name.endswith(".0"):
            return outs[enc_last[int(name.split(".")[1]) - 1]]
        return outs[names[k - 1]]
    return layers, inputs


def _run_generator(prec, off, N, items):
    from wav2lip_b200 import _lib
    ctx = _ctx(prec, off)
    ctx.set_debug(True)
    sd = O.make_state_dict("generator", 0)
    dev = _load(ctx, _lib.NET_GENERATOR, sd)
    mel, face = O.make_generator_inputs(N, seed=2)
    md, fd = mel.cuda().contiguous(), face.cuda().contiguous()
    out = torch.empty((N, 3, 96, 96), device="cuda")
    if prec == F16:
        ctx.f16_overflow(clear=True)
    _lib.check(ctx.lib.w2l_generator_forward(ctx.h, C.c_void_p(md.data_ptr()), C.c_void_p(fd.data_ptr()),
                                             C.c_void_p(out.data_ptr()), N, 0, None))
    torch.cuda.synchronize()
    if prec == F16:
        assert not ctx.f16_overflow(clear=True)
    ks = ctx.plan_kernels(_lib.NET_GENERATOR)
    layers, inputs = _generator_inputs(mel, face, prec)
    outs, worst = _check_chain(ctx, _lib.NET_GENERATOR, layers, sd, inputs, prec, items, f"generator {off or 'all-on'}")
    # output block + fused head: the block output stays fp32 inside the head -> sigmoid(W . relu(block) + b) in float64
    name, row = layers[-1]
    x = inputs(name, outs)[items]
    blk, mag = reference(x, sd, name, row, prec, round_out=False)
    hw = sd["output_block.1.weight"].to("cuda", torch.float64).view(3, 32)
    hb = sd["output_block.1.bias"].to("cuda", torch.float64)
    logit = torch.einsum("oc,nchw->nohw", hw, blk) + hb.view(1, 3, 1, 1)
    ref = torch.sigmoid(logit)
    # |d sigmoid| <= 1/4; the block's fp32 error is <= acc*mag per channel; __expf / division add ~2^-20 absolute
    acc = ACC_X2 if prec == F32X else ACC
    bar = 0.25 * torch.einsum("oc,nchw->nohw", hw.abs(), acc * mag) + 2.0 ** -20
    err = (out[items].double() - ref).abs()
    assert (err <= bar).all(), f"head {off}: max err/bar {(err / bar).max().item():.3g}"
    heads = [k for k in ks if k["head"]]
    assert len(heads) == 1 and heads[0]["family"] == (0 if ("W2L_DISABLE_HALO" in off or prec == F32X) else 1), heads
    return out, ks, worst


@pytest.mark.parametrize("off", NET_SWITCHES, ids=NET_SWITCH_IDS)
@pytest.mark.parametrize("prec", [F16, BF16, F32X], ids=["f16", "bf16", "f32x"])
def test_generator_per_layer(prec, off):
    out, ks, _ = _run_generator(prec, off, 3, slice(None))
    _NET_OUT[(prec, off)] = out
    if prec == F32X:
        assert all(k["family"] == 0 and not k["tma_epi"] and not k["fold"] for k in ks)
    # switches that keep the K order of every output: the network output is bit-identical to all-on
    if off and off[0] in ("W2L_DISABLE_MT2", "W2L_DISABLE_TMAEPI", "W2L_DISABLE_PDL", "W2L_DISABLE_SIDESTREAM"):
        if (prec, ()) not in _NET_OUT:
            _NET_OUT[(prec, ())] = _run_generator(prec, (), 3, slice(None))[0]
        assert torch.equal(out, _NET_OUT[(prec, ())]), off


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_generator_n128_has_mt2_layers(prec):
    """At the serving batch (128 crops) the 32->64 stride-2 encoder block runs two M tiles per CTA."""
    items = [0, 1, 64, 127]
    _out, ks, _ = _run_generator(prec, (), 128, items)
    assert any(k["mt"] == 2 for k in ks), [_short(k) for k in ks]


def _syncnet_disc_check(net_name, prec, off):
    from wav2lip_b200 import _lib
    ctx = _ctx(prec, off)
    ctx.set_debug(True)
    if net_name == "syncnet":
        net, sd = _lib.NET_SYNCNET, O.make_state_dict("syncnet", 0)
        _load(ctx, net, sd)
        mel, face = O.make_syncnet_inputs(4, seed=1)
        md, fd = mel.cuda().contiguous(), face.cuda().contiguous()
        a = torch.empty((4, 512), device="cuda")
        v = torch.empty((4, 512), device="cuda")
        _lib.check(ctx.lib.w2l_syncnet_forward(ctx.h, C.c_void_p(md.data_ptr()), C.c_void_p(fd.data_ptr()),
                                               C.c_void_p(a.data_ptr()), C.c_void_p(v.data_ptr()), 4, None))
        layers = O.syncnet_layers()
        names = [n for n, _ in layers]

        def inputs(name, outs):
            if name == "face_encoder.0":
                return fd
            if name == "audio_encoder.0":
                return md
            return outs[names[names.index(name) - 1]]
    else:
        net, sd = _lib.NET_DISC, O.make_state_dict("disc", 0)
        _load(ctx, net, sd)
        frames = O.make_disc_inputs(2, 5, seed=1).cuda().contiguous()
        prob = torch.empty((10, 1), device="cuda")
        _lib.check(ctx.lib.w2l_disc_forward(ctx.h, C.c_void_p(frames.data_ptr()), C.c_void_p(prob.data_ptr()), 2, 5, None))
        layers = O.disc_layers()
        names = [n for n, _ in layers]
        x0 = torch.cat([frames[:, :, i] for i in range(5)], 0)[:, :, 48:]

        def inputs(name, outs):
            if name == "face_encoder_blocks.0.0":
                return x0
            return outs[names[names.index(name) - 1]]
    torch.cuda.synchronize()
    outs, _ = _check_chain(ctx, net, layers, sd, inputs, prec, slice(None), f"{net_name} {off or 'default'}")
    assert sum(o is not None for o in outs.values()) >= len(layers) - 1
    ks = ctx.plan_kernels(net)
    if off:
        assert all(k["family"] == 0 and k["mt"] == 1 and not k["tma_epi"] and not k["fold"] for k in ks)
    else:
        assert any(k["family"] == 1 for k in ks) and any(k["fold"] for k in ks)


@pytest.mark.parametrize("off", [(), ALL_OFF], ids=["default", "generic-only"])
@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("net_name", ["syncnet", "disc"])
def test_syncnet_disc_per_layer(net_name, prec, off):
    _syncnet_disc_check(net_name, prec, off)
