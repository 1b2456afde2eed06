"""The S3FD network (w2l_s3fd_forward) one op at a time against float64, in every precision and at detector frame sizes.

Every op is checked on the GPU's own export of its input (w2l_set_debug + w2l_debug_layer_output, which exports the 31 conv
layers, then the five max-pools at 31..35 and the three L2Norm outputs at 36..38), so each bar covers one op:
  conv1_1        preprocess(frames) (the caller's fp32 tensor, rounded here as the ingest rounds it)
  conv2_1 ...    the export of the pool before it; other backbone convs the previous conv's export
  heads 0-2      the L2Norm export; heads 3-5 the raw taps (fc7, conv6_2, conv7_2)
Bars (test_gpu_kernel_parity.py defines round16, ulp16, mag and the conv bars, which apply unchanged to the 19 backbone
layers):
  max-pool       bit-exact against a float64 2x2 max-pool of the export, floor semantics at odd sizes.  In F32X the pool
                 compares hi + lo and copies both planes of the winner, which is exact too.
  L2Norm         |y - ref| <= ulp16(max(|y|,|ref|)) + c * 2^-24 * |ref|    (F32X: ulp16(ulp16(max(|y|,|ref|))) in place of
                 the first term: y is stored as hi + lo, and lo is an fp16 rounding of y - hi)
                 c = (C/32 + 5)/2 + 5 = C/64 + 7.5: each lane sums C/32 squares with fmaf and a 5-step butterfly adds the
                 lanes, so the sum of squares (positive terms) carries at most (C/32 + 5) roundings, halved by the sqrt;
                 then one rounding each for the sqrt, the + 1e-10, the reciprocal and the two products.  Not fitted.
  heads          fp32 out through the direct epilogue, no output rounding: |y - ref| <= 2^-16 * mag (F16 / BF16),
                 2^-15 * mag (F32X); the padded channels cout_real..15 are exactly 0.
  12 outputs     bit-identical to the head exports, with the scale-0 max-out (net_s3fd.py:123-126) recomputed in float64.
Each case also runs the forward twice (bit-identical), leaves the fp16 range flag clear at the seeded weights, and pins
the dispatch from w2l_debug_plan_kernels.  W2L_DISABLE_MT2 / _TMAEPI / _PDL keep the 12 maps bit-identical.

Large sizes: images 0 and B-1 are compared.  Layers above 2^17 pixels per image (conv1_x, conv2_x and pools 1-2 at 720p
and 1080p) are compared on a band of rows: the first rows of image 0 and the last rows of image B-1, where the highest
addresses are; each band's reference reads the exported input rows with their halo.  16 x 1080x1920 puts every conv1
activation at 4.2 GB (images 9-15 past 2^31 bytes); 9 x 1080x1920 F32X puts it past 2^31 elements.  One plan is alive at
a time (each case closes its context); a case skips when the card has too little free memory for it.

Measured on one H100 80GB HBM3 (700 W): the 25 tests take 34 s.  Plans (w2l_device_bytes): 16 x 720p 9.5 GiB (F32X
19.2), 16 x 1080p 21.2 GiB, 9 x 1080p F32X 24.3 GiB.  Max-pools bit-exact everywhere.  Max err/bar over the seven sizes:
  op                          f16  bf16   f32x  f16-generic
  conv1_1                    0.98  0.95  0.020  0.98
  conv1_2                    0.94  0.99  0.039  0.94
  conv2_1                    0.93  0.99  0.025  0.93
  conv2_2                    0.93  0.99  0.046  0.93
  conv3_1                    0.90  0.99  0.032  0.90
  conv3_2                    0.90  0.98  0.071  0.90
  conv3_3                    0.90  0.98  0.062  0.89
  conv4_1                    0.90  0.98  0.051  0.90
  conv4_2                    0.90  0.99  0.089  0.89
  conv4_3                    0.88  0.98  0.084  0.89
  conv5_1                    0.83  0.98  0.061  0.84
  conv5_2                    0.86  0.97  0.072  0.86
  conv5_3                    0.89  0.98  0.078  0.89
  fc6                        0.90  0.98  0.805  0.90     (F32X: the border outputs are the bias alone; lo_step bounds them)
  fc7                        0.94  0.99  0.078  0.94
  conv6_1                    0.94  0.99  0.061  0.92
  conv6_2                    0.92  0.98  0.068  0.92
  conv7_1                    0.92  0.98  0.038  0.92
  conv7_2                    0.91  0.99  0.036  0.90
  conv3_3_norm / 4_3 / 5_3   0.50  0.50  0.500  0.50     (the rounding of the output: half of the ulp16 term)
  mbox heads, conf and loc   0.12  0.10  0.088  0.12     (fc7_mbox_loc; the others 0.01-0.06)
Deliberate defects, each caught: a ceil-mode pool (pool2 shape at 150x210), max-out over channel 0 alone (output 0 vs its
head export), the L2Norm weight indexed by lane (conv3_3_norm, err/bar 667), a ReLU on the plain heads
(conv3_3_norm_mbox_conf, 1.2e4), fp32 head outputs rounded to fp16 (conv3_3_norm_mbox_conf, 5.0), and the F32X pool
reading pitch C and the hi plane only (pool1, max |diff| 633), which is what the F32X glue kernels did before they took
the pitch and lo offset.
"""
import ctypes as C
import os
import time

import pytest
import torch
import torch.nn.functional as F

import test_gpu_kernel_parity as P
from oracle import s3fd_oracle as S
from test_gpu_kernel_parity import ACC, ACC_X2, ALL_OFF, BF16, F16, F32X, PREC_NAME, compare, reference, ulp16

pytestmark = pytest.mark.gpu

N_CONV = 31                    # backbone 0..18, heads 19..30
POOL0, NORM0 = N_CONV, N_CONV + 5
BAND = 8                       # output rows compared per band
KEEP = 2 * BAND + 2            # rows kept of a banded export (a pool's band reads 2 * BAND input rows)
BAND_PIXELS = 1 << 17          # exports above this many pixels per image are compared on bands
POOL_AFTER = {1: 0, 3: 1, 6: 2, 9: 3, 12: 4}     # conv layer -> the pool that reads its output
TAP_LAYER = [6, 9, 12, 14, 16, 18]               # conv3_3, conv4_3, conv5_3, fc7, conv6_2, conv7_2
MODES = {"f16": (F16, ()), "bf16": (BF16, ()), "f32x": (F32X, ()), "f16-generic": (F16, ALL_OFF)}
ALL4 = ["f16", "bf16", "f32x", "f16-generic"]
SIZES = [(2, 96, 128, ALL4), (1, 150, 210, ALL4), (3, 32, 32, ALL4), (1, 100, 1000, ALL4), (16, 720, 1280, ALL4),
         (16, 1080, 1920, ["f16", "bf16"]), (9, 1080, 1920, ["f32x"])]
CASES = [(b, h, w, m) for b, h, w, modes in SIZES for m in modes]


# ------------------------------------------------------------------------------------------------------------------
# one context per case, created with the switches in the environment and closed when the case ends
# ------------------------------------------------------------------------------------------------------------------
def _new_ctx(prec, off=()):
    from wav2lip_b200 import _lib
    old = {k: os.environ.get(k) for k in P.FLAGS}
    try:
        for k in P.FLAGS:
            os.environ.pop(k, None)
        for k in off:
            os.environ[k] = "1"
        return _lib.Context(0, prec)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _layers():
    from wav2lip_b200 import _lib
    return _lib.net_layers(_lib.NET_S3FD)


def _plan_bytes(B, H, W, prec):
    """Activation bytes of the S3FD plan of (B, H, W) from its shapes (conv outputs, pools, norms, fp32 heads, input)."""
    planes = 2 if prec == F32X else 1
    a16 = lambda c, hh, ww: B * hh * ww * c * 2 * planes
    tot = a16(16, H, W + 4)   # input (channels padded, a few border columns)
    h, w = H, W
    for li, L in enumerate(_layers()[:19]):
        (kh, kw), (sh, sw), (ph, pw) = L["k"], L["stride"], L["pad"]
        h, w = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
        tot += a16(L["cout"], h, w)
        if li in TAP_LAYER:
            tot += 2 * B * h * w * 16 * 4 + (a16(L["cout"], h, w) if li < 14 else 0)   # two fp32 heads, L2Norm
        if li in POOL_AFTER:
            h, w = h // 2, w // 2
            tot += a16(L["cout"], h, w)
    return tot


def _forward(ctx, frames_u8, sd_dev):
    from wav2lip_b200 import _lib
    B, H, W, _ = frames_u8.shape
    x = S.preprocess(frames_u8).cuda().contiguous()
    dims = (C.c_int32 * 12)()
    _lib.check(ctx.lib.w2l_s3fd_out_dims(H, W, dims))
    outs = []
    for i in range(6):
        for c in (2, 4):
            outs.append(torch.empty((B, c, dims[2 * i], dims[2 * i + 1]), device="cuda", dtype=torch.float32))
    ptrs = (C.c_void_p * 12)(*[o.data_ptr() for o in outs])
    _lib.check(ctx.lib.w2l_s3fd_forward(ctx.h, C.c_void_p(x.data_ptr()), ptrs, B, H, W, None))
    torch.cuda.synchronize()
    return x, outs


def _load(ctx, sd):
    from wav2lip_b200 import _lib
    dev = {k: v.to("cuda", torch.float32).contiguous() for k, v in sd.items()}
    ctx.load_weights(_lib.NET_S3FD, {k: (v.data_ptr(), v.numel()) for k, v in dev.items()})
    torch.cuda.synchronize()
    return dev


# ------------------------------------------------------------------------------------------------------------------
# what is kept of an export: images 0 and B-1 whole, or a band of rows at the top of image 0 and the bottom of image B-1
# ------------------------------------------------------------------------------------------------------------------
class Kept:
    def __init__(self, y):
        B, _, H, W = y.shape
        self.H, self.W = H, W
        self.band = H * W > BAND_PIXELS and H > 2 * KEEP
        if self.band:
            self.top, self.bot = y[:1, :, :KEEP].clone(), y[B - 1:, :, H - KEEP:].clone()
        else:
            self.full = y[sorted({0, B - 1})].clone()


def _top(k, n):
    return k.top[:, :, :n] if k.band else k.full[:1, :, :n]


def _bot(k, n):
    return k.bot[:, :, -n:] if k.band else k.full[-1:, :, -n:]


def _export(ctx, i):
    return P._export(ctx, 3, i)


def _conv_row(L):
    kind = {3: "p", 4: "r"}[L["kind"]]
    return (kind, L["cin"], L["cout_real"] or L["cout"], L["k"], L["stride"], L["pad"], 0, False)


def _check_conv(name, L, xin, yk, sd, prec):
    """Backbone layer: the conv bars of test_gpu_kernel_parity on the kept region; returns max err/bar."""
    row = _conv_row(L)
    sdl = {f"{name}.conv_block.0.weight": sd[name + ".weight"], f"{name}.conv_block.0.bias": sd[name + ".bias"]}
    if not xin.band:
        ref, mag = reference(xin.full, sdl, name, row, prec)
        return compare(yk.full, ref, mag, prec, name)[0]
    assert row[3:6] == ((3, 3), (1, 1), (1, 1)) and (yk.H, yk.W) == (xin.H, xin.W), (name, row)
    worst = 0.0
    rowb = row[:5] + ((0, 1),) + row[6:]         # vertical padding applied to the band by hand
    for x, y, pad in ((_top(xin, BAND + 1), _top(yk, BAND), (0, 0, 1, 0)),
                      (_bot(xin, BAND + 1), _bot(yk, BAND), (0, 0, 0, 1))):
        ref, mag = reference(F.pad(x, pad), sdl, name, rowb, prec)
        worst = max(worst, compare(y, ref, mag, prec, f"{name} band")[0])
    return worst


def _check_pool(k, xin, yk):
    """max-pool k: bit-exact against float64 on the kept region."""
    what = f"pool{k + 1}"
    if not xin.band:
        ref = F.max_pool2d(xin.full.double(), 2, 2)
        y = yk.full.double()
        assert y.shape == ref.shape, (what, tuple(y.shape), tuple(ref.shape))
        assert torch.equal(y, ref), f"{what}: max |diff| {(y - ref).abs().max().item():.3g}"
        return
    Hp = yk.H
    assert Hp == xin.H // 2 and yk.W == xin.W // 2, (what, yk.H, yk.W, xin.H, xin.W)
    lo = 2 * Hp - 2 * BAND - (xin.H - KEEP)      # first input row of the bottom band inside xin.bot
    for x, y in ((xin.top[:, :, :2 * BAND], _top(yk, BAND)), (xin.bot[:, :, lo:lo + 2 * BAND], _bot(yk, BAND))):
        ref = F.max_pool2d(x.double(), 2, 2)
        assert torch.equal(y.double(), ref), f"{what} band: max |diff| {(y.double() - ref).abs().max().item():.3g}"


def _check_l2norm(i, xin, yk, sd, prec):
    """L2Norm i: the bar of the module docstring; returns max err/bar."""
    name = S.TAPS[i]
    assert not xin.band and not yk.band, name
    x = xin.full.double()
    w = sd[name + ".weight"].to("cuda", torch.float64).view(1, -1, 1, 1)
    ref = x / (x.pow(2).sum(1, keepdim=True).sqrt() + 1e-10) * w
    y = yk.full.double()
    assert y.shape == ref.shape and torch.isfinite(y).all(), name
    m = torch.maximum(y.abs(), ref.abs())
    c = x.shape[1] / 64 + 7.5
    bar = (ulp16(ulp16(m, F16), F16) if prec == F32X else ulp16(m, prec)) + c * 2.0 ** -24 * ref.abs()
    r = ((y - ref).abs() / bar).max().item()
    assert r <= 1.0, f"{name} [{PREC_NAME[prec]}]: max err/bar {r:.3g}"
    return r


def _check_head(name, L, xin, y, sd, prec):
    """mbox head: fp32 out, no output rounding; the 16-padded channels are exactly 0.  Returns max err/bar."""
    cr = L["cout_real"]
    assert y.shape[1] == 16 and cr in (2, 4), (name, tuple(y.shape))
    pad = y[:, cr:]
    assert torch.count_nonzero(pad) == 0, f"{name}: padded channels {cr}..15 not zero"
    sdl = {f"{name}.conv_block.0.weight": sd[name + ".weight"], f"{name}.conv_block.0.bias": sd[name + ".bias"]}
    ref, mag = reference(xin.full, sdl, name, _conv_row(L), prec, round_out=False)
    yy = y[:, :cr].double()
    assert yy.shape == ref.shape and torch.isfinite(yy).all(), name
    r = ((yy - ref).abs() / ((ACC_X2 if prec == F32X else ACC) * mag)).max().item()
    assert r <= 1.0, f"{name} [{PREC_NAME[prec]}]: max err/bar {r:.3g}"
    return r


# ------------------------------------------------------------------------------------------------------------------
# dispatch pins
# ------------------------------------------------------------------------------------------------------------------
def _check_dispatch(ks, prec, off, B, H, W):
    by = {}
    for k in ks:
        by.setdefault(k["name"].split(" ")[0].split(".")[0], []).append(k)
    layers = _layers()
    assert set(by) == {L["name"] for L in layers}, sorted(set(by) ^ {L["name"] for L in layers})
    for L in layers[19:]:   # heads: fp32 out through the generic kernel's direct epilogue
        assert all(k["family"] == 0 and not k["tma_epi"] and not k["head"] for k in by[L["name"]]), by[L["name"]]
    if prec == F32X or off:
        assert all(k["family"] == 0 and not k["tma_epi"] and not k["fold"] for k in ks), [P._short(k) for k in ks]
        assert prec == F32X or all(k["mt"] == 1 for k in ks)
        return
    assert all(k["fold"] and k["family"] == 1 for k in by["conv1_1"]), by["conv1_1"]   # K-folded patch kernel
    assert all(k["family"] == 1 and not k["fold"] for k in by["conv1_2"]), by["conv1_2"]
    if H >= 720:
        # conv2_1 .. conv5_3 have enough tiles for BN = 128 (cout is a multiple of 128), and there is no two-M-tile
        # instantiation at BN = 128; where BN drops to 64 there are too few tiles for two per CTA: one M tile throughout
        assert all(k["bn"] == 128 and k["family"] == 0 for L in layers[2:13] for k in by[L["name"]]), \
            [P._short(k) for k in ks]
        assert all(k["mt"] == 1 for k in ks), [P._short(k) for k in ks]


# ------------------------------------------------------------------------------------------------------------------
# the chain
# ------------------------------------------------------------------------------------------------------------------
def _run_case(B, H, W, prec, off):
    from wav2lip_b200 import _lib
    need = _plan_bytes(B, H, W, prec) + B * 64 * H * W * 4 + (4 << 30)
    free, _total = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{free / 2**30:.1f} GiB free on the device, this case needs about {need / 2**30:.1f} GiB")
    t0 = time.time()
    sd = S.make_state_dict(0)
    frames = S.make_images(B, H, W, seed=B + H + W)
    layers = _layers()
    ctx = _new_ctx(prec, off)
    try:
        ctx.set_debug(True)
        _sd_dev = _load(ctx, sd)
        if prec == F16:
            ctx.f16_overflow(clear=True)
        x, outs = _forward(ctx, frames, _sd_dev)
        if prec == F16:
            assert not ctx.f16_overflow(clear=True), "fp16 range flag set at the seeded weights"
        x2, outs2 = _forward(ctx, frames, _sd_dev)
        for i, (a, b) in enumerate(zip(outs, outs2)):
            assert torch.equal(a, b), f"output {i}: two runs differ"
        del x2, outs2
        ks = ctx.plan_kernels(_lib.NET_S3FD)
        plan_bytes = ctx.device_bytes()
        _check_dispatch(ks, prec, off, B, H, W)

        worst, kept = {}, {}
        kept["in"] = Kept(x)
        del x
        for li in range(19):
            name = layers[li]["name"]
            y = _export(ctx, li)
            kept[li] = Kept(y)
            del y
            if li == 0:
                src = kept["in"]
            elif li - 1 in POOL_AFTER:
                src = kept[("pool", POOL_AFTER[li - 1])]
            else:
                src = kept[li - 1]
            worst[name] = _check_conv(name, layers[li], src, kept[li], sd, prec)
            if li in POOL_AFTER:
                k = POOL_AFTER[li]
                y = _export(ctx, POOL0 + k)
                kept[("pool", k)] = Kept(y)
                del y
                _check_pool(k, kept[li], kept[("pool", k)])
                worst[f"pool{k + 1}"] = 0.0
            for old in [k for k in kept if isinstance(k, int) and k < li - 1 and k not in TAP_LAYER]:
                del kept[old]
            torch.cuda.empty_cache()
        heads = []
        for i in range(6):
            src = kept[TAP_LAYER[i]]
            if i < 3:
                y = _export(ctx, NORM0 + i)
                nk = Kept(y)
                del y
                worst[S.TAPS[i]] = _check_l2norm(i, src, nk, sd, prec)
                src = nk
            for h in range(2):
                li = 19 + 2 * i + h
                name = layers[li]["name"]
                y = _export(ctx, li)
                yk = Kept(y)
                del y
                assert not yk.band
                worst[name] = _check_head(name, layers[li], src, yk.full, sd, prec)
                heads.append(yk.full)
        # the 12 module outputs are the head exports; scale 0's conf map is the max-out of its three background logits
        items = sorted({0, B - 1})
        for j, (o, hd) in enumerate(zip(outs, heads)):
            hd = hd.double()
            if j == 0:
                exp = torch.cat([torch.maximum(torch.maximum(hd[:, 0:1], hd[:, 1:2]), hd[:, 2:3]), hd[:, 3:4]], 1)
            else:
                exp = hd[:, : o.shape[1]]
            assert torch.equal(o[items].double(), exp), f"output {j} differs from its head export"
        print(f"\n[s3fd parity] {B}x{H}x{W} {PREC_NAME[prec]}{' generic-only' if off else ''}: plan "
              f"{plan_bytes / 2**30:.2f} GiB (estimate {_plan_bytes(B, H, W, prec) / 2**30:.2f}), "
              f"{time.time() - t0:.1f} s, kernels {sorted({P._short(k) for k in ks})}")
        print("  " + "  ".join(f"{k} {v:.3f}" for k, v in worst.items()))
        return worst
    finally:
        ctx.close()
        torch.cuda.empty_cache()


@pytest.mark.parametrize("case", CASES, ids=[f"{b}x{h}x{w}-{m}" for b, h, w, m in CASES])
def test_s3fd_chain_matches_float64(case):
    B, H, W, mode = case
    prec, off = MODES[mode]
    _run_case(B, H, W, prec, off)


@pytest.mark.parametrize("B,H,W", [(2, 96, 128), (16, 720, 1280)], ids=["2x96x128", "16x720x1280"])
def test_switches_keep_maps_bit_identical(B, H, W):
    """W2L_DISABLE_MT2 / _TMAEPI / _PDL change launches, not the K order of any output: the 12 maps are bit-identical."""
    from wav2lip_b200 import _lib
    sd = S.make_state_dict(0)
    frames = S.make_images(B, H, W, seed=7)
    ref = None
    for off in [(), ("W2L_DISABLE_MT2",), ("W2L_DISABLE_TMAEPI",), ("W2L_DISABLE_PDL",)]:
        ctx = _new_ctx(F16, off)
        try:
            dev = _load(ctx, sd)
            _x, outs = _forward(ctx, frames, dev)
            ks = ctx.plan_kernels(_lib.NET_S3FD)
        finally:
            ctx.close()
        if ref is None:
            ref, ks_on = outs, ks
            continue
        if off == ("W2L_DISABLE_TMAEPI",):
            assert any(k["tma_epi"] for k in ks_on) and not any(k["tma_epi"] for k in ks)
        for i, (a, b) in enumerate(zip(ref, outs)):
            assert torch.equal(a, b), f"{off[0]}: output {i} max diff {(a - b).abs().max().item():.3g}"
    torch.cuda.empty_cache()
