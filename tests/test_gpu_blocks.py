"""Operator-level parity: every distinct conv-block geometry of the three networks through the C-ABI
(w2l_conv_block_forward, via the models.conv mirrors) against the oracle's fp32 CPU block.

Tolerance: the tensor-core path rounds operands to fp16 (10-bit mantissa, the same mantissa as the
TF32 path cuDNN takes for the reference on any Ampere+ GPU) and accumulates in fp32, and the block
output is stored as fp16: one block is therefore exact to ~2^-11 relative to the tensor's magnitude.
The test bar is |err| <= 2e-3 * max|ref| element-wise."""
import pytest
import torch

from oracle import w2l_oracle as O

pytestmark = pytest.mark.gpu

REL = 2e-3

# name, kind, cin, cout, k, stride, pad, out_pad, residual, N, H, W
CASES = [
    ("gen 3x3 64 res", "c", 64, 64, 3, 1, 1, 0, True, 2, 24, 24),
    ("gen 3x3 64 96x96", "c", 64, 64, 3, 1, 1, 0, True, 1, 96, 96),
    ("gen 3x3 64 96x96 res N=5", "c", 64, 64, 3, 1, 1, 0, True, 5, 96, 96),
    ("3x3 64 lrelu 32x64", "n", 64, 64, 3, 1, 1, 0, False, 19, 32, 64),
    ("gen 1x1 512", "c", 512, 512, 1, 1, 0, 0, False, 5, 1, 1),
    ("gen 3x3 32 res (64B swizzle)", "c", 32, 32, 3, 1, 1, 0, True, 2, 48, 48),
    ("gen 16->32 s2 (32B swizzle)", "c", 16, 32, 3, 2, 1, 0, False, 2, 96, 96),
    ("gen 7x7 6->16", "c", 6, 16, 7, 1, 3, 0, False, 2, 96, 96),
    ("gen 7x7 6->16 N=5", "c", 6, 16, 7, 1, 3, 0, False, 5, 96, 96),
    ("gen 3x3 128 res", "c", 128, 128, 3, 1, 1, 0, True, 3, 12, 12),
    ("gen 3x3 256 res", "c", 256, 256, 3, 1, 1, 0, True, 3, 6, 6),
    ("gen 3x3 384 res", "c", 384, 384, 3, 1, 1, 0, True, 2, 12, 12),
    ("gen 3x3 512 res 3x3", "c", 512, 512, 3, 1, 1, 0, True, 3, 3, 3),
    ("gen 64->128 s2", "c", 64, 128, 3, 2, 1, 0, False, 2, 24, 24),
    ("audio s(3,1)", "c", 32, 64, 3, (3, 1), 1, 0, False, 2, 80, 16),
    ("audio s3", "c", 64, 128, 3, 3, 1, 0, False, 2, 27, 16),
    ("audio s(3,2)", "c", 128, 256, 3, (3, 2), 1, 0, False, 2, 9, 6),
    ("3x3 pad0 -> 1x1", "c", 512, 512, 3, 1, 0, 0, False, 3, 3, 3),
    ("audio 1->32", "c", 1, 32, 3, 1, 1, 0, False, 2, 80, 16),
    ("output 80->32", "c", 80, 32, 3, 1, 1, 0, False, 1, 96, 96),
    ("convT 1x1->3x3 (GEMM form)", "t", 1024, 512, 3, 1, 0, 0, False, 3, 1, 1),
    ("convT s2 1024->512", "t", 1024, 512, 3, 2, 1, 1, False, 2, 3, 3),
    ("convT s2 768->384", "t", 768, 384, 3, 2, 1, 1, False, 1, 6, 6),
    ("convT s2 320->128", "t", 320, 128, 3, 2, 1, 1, False, 1, 24, 24),
    ("convT s2 160->64", "t", 160, 64, 3, 2, 1, 1, False, 1, 48, 48),
    ("sync 7x7 15->32", "c", 15, 32, 7, 1, 3, 0, False, 2, 48, 96),
    ("sync k5 s(1,2) p1 -> 46x47", "c", 32, 64, 5, (1, 2), 1, 0, False, 2, 48, 96),
    ("sync 46x47 res", "c", 64, 64, 3, 1, 1, 0, True, 2, 46, 47),
    ("sync 46x47 s2 -> 23x24", "c", 64, 128, 3, 2, 1, 0, False, 2, 46, 47),
    ("sync 23x24 res", "c", 128, 128, 3, 1, 1, 0, True, 2, 23, 24),
    ("disc 7x7 3->32 lrelu", "n", 3, 32, 7, 1, 3, 0, False, 2, 48, 96),
    ("disc 7x7 3->32 lrelu N=9", "n", 3, 32, 7, 1, 3, 0, False, 9, 48, 96),
    ("disc k5 s(1,2)", "n", 32, 64, 5, (1, 2), 2, 0, False, 2, 48, 96),
    ("disc k5", "n", 64, 64, 5, 1, 2, 0, False, 2, 48, 48),
    ("disc k5 s2", "n", 128, 256, 5, 2, 2, 0, False, 2, 24, 24),
    ("disc k5 256", "n", 256, 256, 5, 1, 2, 0, False, 1, 12, 12),
    # edge cases: batch of one, ragged sizes that do not fill a 128-row tile, odd extents
    ("N=1 1x1", "c", 512, 512, 1, 1, 0, 0, False, 1, 1, 1),
    ("ragged 5x7", "c", 64, 64, 3, 1, 1, 0, True, 3, 5, 7),
    ("ragged 13x11 s2", "c", 32, 64, 3, 2, 1, 0, False, 5, 13, 11),
    ("N=131 3x3 spatial", "c", 64, 64, 3, 1, 1, 0, True, 131, 3, 3),
    # batches large enough for many 128-row tiles per SM at 128-channel tiles:
    # residual, three channel tiles, ragged boxes, strided, transposed-conv phases
    ("large N 3x3 128 res 24x24 N=140", "c", 128, 128, 3, 1, 1, 0, True, 140, 24, 24),
    ("large N 3x3 384 res 12x12 N=190", "c", 384, 384, 3, 1, 1, 0, True, 190, 12, 12),
    ("large N ragged 23x24 128 res N=150", "c", 128, 128, 3, 1, 1, 0, True, 150, 23, 24),
    ("large N 64->128 s2 48x48 N=140", "c", 64, 128, 3, 2, 1, 0, False, 140, 48, 48),
    ("large N convT s2 320->128 N=150", "t", 320, 128, 3, 2, 1, 1, False, 150, 24, 24),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_block_matches_oracle(case):
    from wav2lip_b200.models.conv import Conv2d, Conv2dTranspose, nonorm_Conv2d
    _name, kind, cin, cout, k, s, p, op, res, N, H, W = case
    g = torch.Generator().manual_seed(1234)
    row = (kind, cin, cout, k, s, p, op, res)
    sd = O._block_tensors("b", row, g, 1.0)
    x = torch.rand((N, cin, H, W), generator=g) * 2 - 0.5
    with torch.no_grad():
        ref = O.block_forward(x, sd, "b", row)
    if kind == "t":
        m = Conv2dTranspose(cin, cout, k, s, p, op)
    elif kind == "n":
        m = nonorm_Conv2d(cin, cout, k, s, p)
    else:
        m = Conv2d(cin, cout, k, s, p, residual=res)
    m.load_state_dict({kk[2:]: v for kk, v in sd.items()}, strict=True)
    m = m.cuda().eval()
    with torch.no_grad():
        y = m(x.cuda())
    torch.cuda.synchronize()
    assert tuple(y.shape) == tuple(ref.shape)
    err = (y.cpu() - ref).abs().max().item()
    assert err <= REL * ref.abs().max().item(), f"max|err| {err:.4g} vs max|ref| {ref.abs().max().item():.4g}"


# Block descriptions the C ABI's single-block entries must refuse before they allocate or launch anything:
# (what is wrong, kind, cin, cout, kh, kw, sh, sw, ph, pw, residual), applied to a (1, cin, 8, 8) input
BAD_LAYERS = [
    ("stride 0", 0, 64, 64, 3, 3, 0, 1, 1, 1, 0),
    ("8x8 kernel", 0, 64, 64, 8, 8, 1, 1, 3, 3, 0),
    ("residual with cin != cout", 0, 32, 64, 3, 3, 1, 1, 1, 1, 1),
]


def bad_layer_calls():
    """(what, LayerInfo, tensors) per BAD_LAYERS row; the tensors are large enough for any shape the row implies."""
    from wav2lip_b200 import _lib
    for what, kind, cin, cout, kh, kw, sh, sw, ph, pw, res in BAD_LAYERS:
        li = _lib.LayerInfo()
        li.name = b"block"
        li.kind, li.cin, li.cout, li.kh, li.kw, li.sh, li.sw, li.ph, li.pw, li.out_pad, li.residual = (
            kind, cin, cout, kh, kw, sh, sw, ph, pw, 0, res)
        t = {"x": torch.zeros(1, cin, 8, 8, device="cuda"), "w": torch.zeros(cout, cin, kh, kw, device="cuda"),
             "y": torch.zeros(1, cout, 16, 16, device="cuda")}
        t.update({k: torch.ones(cout, device="cuda") for k in ("b", "gamma", "beta", "mean", "var")})
        yield what, li, t


def test_block_rejects_bad_arguments():
    import ctypes as C

    from wav2lip_b200 import _lib
    from wav2lip_b200.models.conv import Conv2d
    m = Conv2d(64, 64, 3, 1, 1).eval()  # parameters on the CPU
    with pytest.raises(_lib.W2LError):
        m(torch.zeros(1, 64, 8, 8))      # CPU input: no fallback
    m = Conv2d(64, 24, 3, 1, 1).cuda().eval()  # cout not a multiple of 16 is outside the kernel family
    with pytest.raises(_lib.W2LError):
        m(torch.zeros(1, 64, 8, 8, device="cuda"))
    m = Conv2d(64, 64, 3, 1, 1).cuda()   # train mode: batch-stat BN is not built
    with pytest.raises(NotImplementedError):
        m(torch.zeros(1, 64, 8, 8, device="cuda"))
    ctx = _lib.Context(0, _lib.PREC_F16)
    P = lambda a: C.c_void_p(a.data_ptr())
    for what, li, t in bad_layer_calls():
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.W2LError):
            _lib.check(ctx.lib.w2l_conv_block_forward(ctx.h, C.byref(li), P(t["x"]), 1, 8, 8, P(t["w"]), P(t["b"]),
                                                      P(t["gamma"]), P(t["beta"]), P(t["mean"]), P(t["var"]), P(t["y"]),
                                                      None))
        assert ctx.launch_count() == n0, what
