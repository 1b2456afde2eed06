"""The generic conv kernel's two consumer warpgroups (conv_igemm.cuh, MT = 1): warpgroup g takes the CTA's tiles g, g+2, ...
and finds its ring slots from the CTA-global K-step index, and the two K loops hand over to each other through a pair of
named barriers.  These cases give every CTA several tiles, with K-step counts that wrap the ring out of step with the tile
boundaries (1, 2, 3, 18, 27 steps against 5- or 8-stage rings), odd tile counts per CTA, and launches with between 132
and 264 tiles where most CTAs leave warpgroup 1 without a tile.  Every case is compared with the float64 reference of
test_gpu_kernel_parity.py at its bars, in fp16 and bf16, runs twice with bit-identical results and asserts the kernel
that ran; the residual cases also run with the direct epilogue (W2L_DISABLE_TMAEPI, bit-identical to the staged one) and
in the split-operand mode.  The fused generator head runs on the generic kernel with W2L_DISABLE_HALO at N=8.
"""

import pytest
import torch

import test_gpu_kernel_parity as P
from test_gpu_kernel_parity import BF16, F16, F32X, _c

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _close_contexts():
    yield
    for c in P._CTX.values():
        c.close()
    P._CTX.clear()


# (name, row, N, H, W, expected kernel, tiles per launch)
CASES = [
    ("pp BN128 BK64 k_steps=1 1x1 N=76800", _c(64, 128, 1, 1, 0), 76800, 1, 1, "I128.64e", 600),
    ("pp BN128 BK64 k_steps=3 odd tiles per CTA 1x1 N=50816", _c(192, 128, 1, 1, 0), 50816, 1, 1, "I128.64e", 397),
    ("pp BN128 res two passes k_steps=2 150 tiles", _c(128, 128, 1, 1, 0, True), 2100, 3, 3, "I128.64e", 150),
    ("pp BN128 res 3x3 k_steps=18 24x24 N=64", _c(128, 128, 3, 1, 1, True), 64, 24, 24, "I128.64e", 288),
    ("pp BN128 BK16 k_steps=3 1x1 N=67968", _c(48, 128, 1, 1, 0), 67968, 1, 1, "I128.16e", 531),
    ("pp BN128 BK32 3x3 k_steps=27 48x48 N=16", _c(96, 128, 3, 1, 1), 16, 48, 48, "I128.32e", 288),
    ("pp BN64 BK16 1x1 48->192 N=25600", _c(48, 192, 1, 1, 0), 25600, 1, 1, "I64.16e", 600),
    ("pp BN32 BK16 3x3 48->96 24x24 N=24", _c(48, 96, 3, 1, 1), 24, 24, 24, "I32.16e", 324),
]
IDS = [c[0] for c in CASES]
RES_CASES = [c for c in CASES if c[1][7]]


def _tiles(k):
    return ((k["m_tiles"] + k["mt"] - 1) // k["mt"]) * k["n_tiles"]


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_pingpong_matches_float64(case, prec):
    name, row, N, H, W, expect, tiles = case
    ks = P.run_case((name, row, N, H, W, expect), prec)["kernels"]
    assert len(ks) == 1 and ks[0]["mt"] == 1, ks
    assert _tiles(ks[0]) == tiles and ks[0]["grid"] < tiles, ks[0]


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", RES_CASES, ids=[c[0] for c in RES_CASES])
def test_pingpong_direct_epilogue_is_bit_identical(case, prec):
    name, row, N, H, W, expect, tiles = case
    off = ("W2L_DISABLE_TMAEPI",)
    P.run_case((name, row, N, H, W, expect), prec)
    ks = P.run_case((name, row, N, H, W, expect), prec, off)["kernels"]
    assert len(ks) == 1 and not ks[0]["tma_epi"] and ks[0]["family"] == 0 and _tiles(ks[0]) == tiles, ks
    sd, x = P._tensors(row, 1234, N, H, W)
    y_on = P.block_forward(P._ctx(prec), row, x, sd)
    y_off = P.block_forward(P._ctx(prec, off), row, x, sd)
    assert torch.equal(y_on, y_off), f"{name}: staged and direct epilogues differ by {(y_on - y_off).abs().max().item():.3g}"


@pytest.mark.parametrize("case", RES_CASES, ids=[c[0] for c in RES_CASES])
def test_pingpong_f32x(case):
    name, row, N, H, W, expect, _tiles_ = case
    ks = P.run_case((name, row, N, H, W, expect), F32X)["kernels"]
    assert all(k["family"] == 0 and not k["tma_epi"] and k["grid"] < _tiles(k) for k in ks), ks


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_pingpong_generic_head_n8(prec):
    """The fused 1x1 + sigmoid head on the generic kernel (HALO off) at N=8: 576 tiles of the 96x96 output block."""
    off = ("W2L_DISABLE_HALO",)
    out, ks, _ = P._run_generator(prec, off, 8, slice(None))
    heads = [k for k in ks if k["head"]]
    assert len(heads) == 1 and heads[0]["family"] == 0 and heads[0]["grid"] < _tiles(heads[0]), heads
    out2, _, _ = P._run_generator(prec, off, 8, slice(None))
    assert torch.equal(out, out2), "generator output differs between two runs"
