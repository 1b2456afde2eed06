"""The channel-major form of the generic kernel (conv_igemm_kernel<128, 64, ., ., 1, true>: 128 output channels on wgmma's M,
one warpgroup per 64-channel half, a box of 256 output pixels on N) against float64 with the kernel's rounding points, at
the bars of test_gpu_kernel_parity.py (|y - ref| <= ulp16 + 2^-16 * mag, mean rounding bias within 0.05 ulp), in fp16
and bf16.

Every case asserts that the launch ran in that form (its plan label ends in "[cm]"), runs twice with bit-identical
results and leaves the fp16 range flag clear.  The geometries cover 128, 256 and 384 channels with and without a
residual, a ragged box that leaves some of the 256 GEMM columns outside the box and some box pixels outside the image,
CTAs with an odd number of tiles, a launch with fewer tiles than CTAs, and the decoder blocks that store into a channel
slice of a concat buffer.  The phase launches of a stride-2 transposed conv (strided, interleaved output) stay row-major.
The form keeps the K order of every output, so its results are also compared bit for bit with the row-major kernel
(W2L_DISABLE_TMAEPI turns the staged epilogue, and with it the form, off).
"""
import pytest
import torch

import test_gpu_kernel_parity as P
from test_gpu_kernel_parity import BF16, F16, _c, _n, _p, _t

pytestmark = pytest.mark.gpu

CM = "[cm]"

# (name, row, N, H, W, expected short name of every launch ("*" = not asserted))
CASES = [
    ("128 res 48x48 N=160", _c(128, 128, 3, 1, 1, True), 160, 48, 48, "I128.64e"),
    ("128 relu 48x48 N=160", _c(128, 128, 3, 1, 1), 160, 48, 48, "I128.64e"),
    ("256 res 24x24 N=320", _c(256, 256, 3, 1, 1, True), 320, 24, 24, "I128.64e"),
    ("256 lrelu 24x24 N=320", _n(256, 256, 3, 1, 1), 320, 24, 24, "I128.64e"),
    ("384 res 12x12 N=1408", _c(384, 384, 3, 1, 1, True), 1408, 12, 12, "I128.64e"),
    ("384 plain 12x12 N=1408", _p(384, 384, 3, 1, 1), 1408, 12, 12, "I128.64e"),
    # 9 x 7 x 4 boxes: 252 of the 256 GEMM columns, and the last box row of every image ragged (61 = 8 x 7 + 5)
    ("ragged 61x45 res N=32", _c(128, 128, 3, 1, 1, True), 32, 61, 45, "I128.64e"),
    # 396 tiles = 3 per CTA on 132 SMs
    ("odd tiles per CTA 48x48 N=44 res", _c(128, 128, 3, 1, 1, True), 44, 48, 48, "I128.64e"),
    # 108 tiles of 54 K steps: some CTAs have none
    ("fewer tiles than CTAs 384 12x12 N=64 res", _c(384, 384, 3, 1, 1, True), 64, 12, 12, "I128.64e"),
]
IDS = [c[0] for c in CASES]
CONVT = ("convT s2 512->256 24x24 N=320", _t(512, 256, 3, 2, 1, 1), 320, 24, 24, "*")


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in P._CTX.values():
        c.close()
    P._CTX.clear()


def _is_cm(k):
    return k["name"].endswith(CM)


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_chmajor_matches_float64(case, prec):
    ks = P.run_case(case, prec)["kernels"]
    assert len(ks) == 1 and _is_cm(ks[0]), ks


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_convt_phases_stay_row_major(prec):
    """The phase launches of a stride-2 transposed conv store every second pixel of every second row: they keep the
    row-major tiles (the interleaved stores did not gain in the channel-major form) and match float64."""
    ks = P.run_case(CONVT, prec)["kernels"]
    assert len(ks) == 4 and not any(_is_cm(k) for k in ks), [k["name"] for k in ks]


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", [CASES[0], CASES[2], CASES[6], CASES[8]], ids=[CASES[i][0] for i in (0, 2, 6, 8)])
def test_chmajor_bit_identical_to_row_major(case, prec):
    name, row, N, H, W, _e = case
    sd, x = P._tensors(row, 1234, N, H, W)
    off = ("W2L_DISABLE_TMAEPI",)
    y_cm = P.block_forward(P._ctx(prec), row, x, sd)
    assert _is_cm(P._ctx(prec).plan_kernels(-1)[0])
    y_rm = P.block_forward(P._ctx(prec, off), row, x, sd)
    k_rm = P._ctx(prec, off).plan_kernels(-1)[0]
    assert not _is_cm(k_rm) and not k_rm["tma_epi"], k_rm
    assert torch.equal(y_cm, y_rm), f"{name}: max diff {(y_cm - y_rm).abs().max().item():.3g}"


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_chmajor_channel_slice_destination(prec):
    """At N=160 the 128-channel 48x48 decoder blocks run channel-major; face_decoder_blocks.5.2 stores into its channel
    slice of the concat buffer that feeds the next block.  Every block is checked against float64 on the GPU's own
    export of its input (items 0, 1, 80, 159), and the network runs twice with bit-identical results."""
    items = [0, 1, 80, 159]
    out, ks, _worst = P._run_generator(prec, (), 160, items)
    for name in ("face_decoder_blocks.5.1", "face_decoder_blocks.5.2"):
        got = [k for k in ks if k["name"].split(" ")[0] == name]
        assert len(got) == 1 and _is_cm(got[0]), (name, got)
    out2, _ks, _w = P._run_generator(prec, (), 160, items)
    assert torch.equal(out, out2)


def test_chmajor_every_instantiation_covered():
    """Every instantiation that has the channel-major form met float64 in that form, in fp16 and in bf16."""
    from wav2lip_b200 import _lib
    table = {(k["bn"], k["bk"], k["bf16"]) for k in _lib.kernel_table() if k["family"] == 0 and k["name"] == CM}
    assert table == {(128, 64, 0), (128, 64, 1)}, table
    seen = set()
    for prec in (F16, BF16):
        for case in CASES:
            seen |= {(k["bn"], k["bk"], k["bf16"]) for k in P.run_case(case, prec)["kernels"] if _is_cm(k)}
    assert table <= seen, table - seen


def test_chmajor_range_flag_ignores_pixels_outside_the_image():
    """Channel 0 = 80000 - 32 * (in-image taps x 128 input channels of 1): at least 4 taps inside the image (a corner)
    keeps every stored pixel <= 63616, but the pixels of the ragged 9 x 7 x 4 boxes below the bottom edge see 0..3
    taps and exceed 65504, and the 4 GEMM columns past the 252-pixel box hold stale rows.  They are never stored
    and must not raise the flag.  (All values are exact in fp16.)"""
    N, H, W = 32, 61, 45
    w = torch.zeros(128, 128, 3, 3)
    w[0] = -32.0
    b = torch.zeros(128)
    b[0] = 80000.0
    x = torch.ones(N, 128, H, W)
    ctx = P._ctx(F16)
    row = _p(128, 128, 3, 1, 1)
    sd = {"b.conv_block.0.weight": w, "b.conv_block.0.bias": b}
    ctx.f16_overflow(clear=True)
    y = P.block_forward(ctx, row, x, sd)
    flag = ctx.f16_overflow(clear=True)
    ks = ctx.plan_kernels(-1)
    assert len(ks) == 1 and _is_cm(ks[0]), ks
    assert not flag
    taps = torch.ones(1, 1, H, W)
    taps = torch.nn.functional.conv2d(torch.nn.functional.pad(taps, (1, 1, 1, 1)), torch.ones(1, 1, 3, 3))[0, 0]
    expect = (80000.0 - 32.0 * 128.0 * taps).to(y.device)
    assert torch.equal(y[:, 0], expect.expand(N, H, W)), (y[0, 0] - expect).abs().max().item()
    assert torch.equal(y[:, 1:], torch.zeros_like(y[:, 1:]))


def test_chmajor_range_flag_one_element():
    """y = x[channel 0] + 6016 on output channel 0 (centre tap only): one input of 60000 makes one output 66016 > 65504,
    which sets the flag; with 59008 the output is 65024 and the flag stays clear."""
    N, H, W = 32, 61, 45
    w = torch.zeros(128, 128, 3, 3)
    w[0, 0, 1, 1] = 1.0
    b = torch.zeros(128)
    b[0] = 6016.0
    ctx = P._ctx(F16)
    row = _p(128, 128, 3, 1, 1)
    sd = {"b.conv_block.0.weight": w, "b.conv_block.0.bias": b}
    for v, over in ((59008.0, False), (60000.0, True)):
        x = torch.zeros(N, 128, H, W)
        x[5, 0, 33, 20] = v
        ctx.f16_overflow(clear=True)
        y = P.block_forward(ctx, row, x, sd)
        flag = ctx.f16_overflow(clear=True)
        assert _is_cm(ctx.plan_kernels(-1)[0])
        assert flag == over, (v, flag)
        expect = torch.full((H, W), 6016.0, device=y.device)
        expect[33, 20] = float("inf") if over else v + 6016.0
        assert torch.equal(y[5, 0], expect), (v, y[5, 0, 33, 19:23].tolist())
