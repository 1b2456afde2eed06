"""The channel-major form of the patch kernel (conv_patch_kernel<64, 64>: 64 output channels on wgmma's M, an 8 x 32
tile of 256 pixels on N) against float64 with the kernel's rounding points, at the bars of test_gpu_kernel_parity.py
(|y - ref| <= ulp16 + 2^-16 * mag, mean rounding bias within 0.05 ulp), in fp16 and bf16.

Every case asserts that the launch ran on that kernel (w2l_debug_plan_kernels), runs twice with bit-identical results
and leaves the fp16 range flag clear.  The geometries aim at the parts of the form the network layers do not all reach:
ragged tiles in both directions with an odd width (the last column pair of a row straddles the image edge), CTAs with an
odd number of tiles, a launch with fewer tiles than CTAs (the second consumer warpgroup has no tile), the residual and
the plain form, each activation, and a destination whose pixel pitch is wider than the 64 channels it stores.
"""
import pytest
import torch

import test_gpu_kernel_parity as P
from oracle import w2l_oracle as O
from test_gpu_kernel_parity import BF16, F16, _c, _n, _p

pytestmark = pytest.mark.gpu

CHMAJOR = "P64.64"

CASES = [
    ("ragged 61x45 res", _c(64, 64, 3, 1, 1, True), 2, 61, 45, CHMAJOR),
    ("ragged 61x45 relu", _c(64, 64, 3, 1, 1), 2, 61, 45, CHMAJOR),
    ("lrelu 40x40", _n(64, 64, 3, 1, 1), 2, 40, 40, CHMAJOR),
    ("no activation 46x47", _p(64, 64, 3, 1, 1), 2, 46, 47, CHMAJOR),
    # 324 tiles: on any GPU with fewer SMs, some CTAs take an odd number of tiles
    ("odd tiles per CTA 96x96 N=9 res", _c(64, 64, 3, 1, 1, True), 9, 96, 96, CHMAJOR),
    # 5 tiles, one per CTA: the second consumer warpgroup of every CTA has none
    ("one tile per CTA 32x40 res", _c(64, 64, 3, 1, 1, True), 1, 32, 40, CHMAJOR),
]


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in P._CTX.values():
        c.close()
    P._CTX.clear()


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_chmajor_matches_float64(case, prec):
    P.run_case(case, prec)


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_chmajor_channel_slice_destination(prec):
    """face_decoder_blocks.6.2 stores its 64 channels into the 80-channel concat buffer of the output block: the
    generator checked layer by layer (every block against float64 on the GPU's own export of its input), twice."""
    from wav2lip_b200 import _lib
    names = [n for n, _ in O.generator_layers()]
    i62 = names.index("face_decoder_blocks.6.2")
    runs = []
    for _ in range(2):
        out, ks, _worst = P._run_generator(prec, (), 3, slice(None))
        runs.append((out, P._export(P._ctx(prec), _lib.NET_GENERATOR, i62)))
    for name in ("face_decoder_blocks.6.1", "face_decoder_blocks.6.2"):
        got = [P._short(k) for k in ks if k["name"].split(" ")[0] == name]
        assert got == [CHMAJOR], (name, got)
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def _plain_block(w, b, x, prec):
    """One 64 -> 64 3x3 plain (no BatchNorm, no activation) block on a fresh fp16 range flag: (output, flag)."""
    ctx = P._ctx(prec)
    row = _p(64, 64, 3, 1, 1)
    sd = {"b.conv_block.0.weight": w, "b.conv_block.0.bias": b}
    ctx.f16_overflow(clear=True)
    y = P.block_forward(ctx, row, x, sd)
    flag = ctx.f16_overflow(clear=True)
    ks = [P._short(k) for k in ctx.plan_kernels(-1)]
    assert ks == [CHMAJOR], ks
    return y, flag


def test_chmajor_range_flag_one_element():
    """y = x[channel 0] + 6016 on channel 0 (centre tap only): one input of 60000 makes one output 66016 > 65504, which
    sets the flag; its neighbour in the same packed pair (even column, so the pair is this pixel and the next) stays
    6016.  With 59008 the output is 65024 and the flag stays clear.  (All values are exact in fp16.)"""
    N, H, W = 1, 61, 45
    w = torch.zeros(64, 64, 3, 3)
    w[0, 0, 1, 1] = 1.0
    b = torch.zeros(64)
    b[0] = 6016.0
    for v, over in ((59008.0, False), (60000.0, True)):
        x = torch.zeros(N, 64, H, W)
        x[0, 0, 33, 20] = v
        y, flag = _plain_block(w, b, x, F16)
        assert flag == over, (v, flag)
        expect = torch.full((H, W), 6016.0, device=y.device)
        expect[33, 20] = float("inf") if over else v + 6016.0
        assert torch.equal(y[0, 0], expect), (v, y[0, 0, 33, 19:23].tolist())


def test_chmajor_range_flag_ignores_pixels_outside_the_image():
    """Channel 0 = 72000 - 32 * (number of in-image taps x 64 input channels of 1): at least 4 taps inside the image
    (a corner) keeps every stored pixel <= 63808, but the tile's pixels beyond the right and bottom edges see 0..3 taps
    and exceed 65504.  W is odd, so the last column pair of each row straddles the edge.  They are never stored and
    must not raise the flag."""
    N, H, W = 2, 61, 45
    w = torch.zeros(64, 64, 3, 3)
    w[0] = -32.0
    b = torch.zeros(64)
    b[0] = 72000.0
    x = torch.ones(N, 64, H, W)
    y, flag = _plain_block(w, b, x, F16)
    assert not flag
    taps = torch.ones(1, 1, H, W)
    taps = torch.nn.functional.conv2d(torch.nn.functional.pad(taps, (1, 1, 1, 1)), torch.ones(1, 1, 3, 3))[0, 0]
    expect = (72000.0 - 32.0 * 64.0 * taps).to(y.device)
    assert torch.equal(y[:, 0], expect.expand(N, H, W)), (y[0, 0] - expect).abs().max().item()
    assert torch.equal(y[:, 1:], torch.zeros_like(y[:, 1:]))
