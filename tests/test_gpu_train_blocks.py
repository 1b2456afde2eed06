"""Training row (SURVEY.md section 8 f1), operator level: one conv.py block in TRAIN mode — forward on batch statistics
and the full backward (dx via the dgrad launches, dW via the wgmma wgrad kernel + split-K reduction, dgamma / dbeta /
dbias, running-average update) — through the C-ABI entry `w2l_conv_block_train`, for every distinct block geometry of
the three networks, against oracle/backward_recipe.py (float64; itself equal to torch autograd, tests/
test_backward_recipe.py).

Two bars per case:
  * SAME ROUNDING POINTS (the parity bar, DESIGN.md section 7): the reference below is the float64 recipe with the
    kernels' own rounding points — bf16 operands (x, w, dy), z stored in bf16 before the statistics, y / dz / du stored in
    bf16 — so what remains is fp32-vs-fp64 accumulation and the rare 1-ulp bf16 rounding flip: relative L2 <= 5e-3 on
    y, dx, dW, dgamma, dbeta, dbias.
  * EXACT OPERANDS (information, loose): against the unrounded float64 recipe the same tensors differ by 3-9 % — the
    ReLU / LeakyReLU mask of the ~0.2 % of pre-activations that sit within bf16 rounding of zero flips, and a flipped
    element carries a full-size error (tests/test_precision_model.py measures the same 3 % on the CPU); asserted <= 0.15."""
import ctypes as C

import pytest
import torch

from oracle import backward_recipe as R
from oracle import w2l_oracle as O

pytestmark = pytest.mark.gpu

REL = 5e-3       # same rounding points
LOOSE = 0.15     # exact operands


def bf16(t):
    return t.to(torch.bfloat16).to(torch.float64)


def reference_same_rounding(x, w, b, gamma, beta, dy, row):
    """float64 block forward / backward with the kernels' rounding points (see the module docstring)."""
    kind, _cin, _cout, k, s, p, op, res = row
    F = torch.nn.functional
    xq, wq, dyq = bf16(x), bf16(w), bf16(dy)
    if kind == "t":
        z = F.conv_transpose2d(xq, wq, None, stride=O._pair(s), padding=O._pair(p), output_padding=O._pair(op))
    else:
        z = F.conv2d(xq, wq, None, stride=O._pair(s), padding=O._pair(p))
    if kind == "n":
        y = bf16(F.leaky_relu(z + b.double()[None, :, None, None], 0.01))
        dz = bf16(dyq * torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.01)))
        out = {"y": y, "db": dz.sum(dim=(0, 2, 3)), "dgamma": None, "dbeta": None}
        du = None
    else:
        zr = bf16(z)                                        # the conv epilogue stores z in bf16; the bias never enters
        mean = zr.mean(dim=(0, 2, 3))
        var = zr.var(dim=(0, 2, 3), unbiased=False)
        invstd = (var + 1e-5).rsqrt()
        zhat = (zr - mean[None, :, None, None]) * invstd[None, :, None, None]
        u = zhat * gamma.double()[None, :, None, None] + beta.double()[None, :, None, None]
        if res:
            u = u + xq
        y = bf16(F.relu(u))
        du = dyq * (y > 0).to(torch.float64)
        m = du.numel() / du.shape[1]
        dbeta = du.sum(dim=(0, 2, 3))
        dgamma = (du * zhat).sum(dim=(0, 2, 3))
        dz = bf16((gamma.double() * invstd)[None, :, None, None] * (du - dbeta[None, :, None, None] / m - zhat * dgamma[None, :, None, None] / m))
        out = {"y": y, "dgamma": dgamma, "dbeta": dbeta, "db": None, "zmean": mean, "zvar": var}
    dx = R.conv_dgrad(dz, wq, row, (x.shape[2], x.shape[3]))
    if kind != "n" and res:
        dx = dx + bf16(du)
    out["dx"] = dx
    out["dw"] = R.conv_wgrad(xq, dz, row)
    return out


def rel_l2(got, ref):
    return ((got.double() - ref.double()).norm() / (ref.double().norm() + 1e-30)).item()


def _cases():
    rows, seen = [], set()
    allr = [r for _, r in O.generator_layers()] + [r for _, r in O.syncnet_layers()] + [r for _, r in O.disc_layers()]
    for r in allr:
        key = (r[0], O._pair(r[3]), O._pair(r[4]), O._pair(r[5]), r[6], r[7])
        if key not in seen:
            seen.add(key)
            rows.append(r)
    out = []
    for r in rows:                      # every distinct geometry with moderate channel counts
        kind, cin, cout, k, s, p, op, res = r
        cin2 = min(cin, 48)
        cout2 = cin2 if res else min(cout, 32)
        if res:
            cin2 = cout2 = 32
        out.append(((kind, cin2, cout2, k, s, p, op, res), 2, (12, 13)))
    # real channel counts that exercise every wgrad tile shape (N tiles of 16/32/64/128/256, several M tiles, tap groups)
    out += [
        (O._c(6, 16, 7, 1, 3), 2, (24, 24)),            # first block: Cin 6 (padded to 16), 49 taps in two groups
        (O._c(64, 64, 3, 1, 1, True), 2, (24, 24)),      # the 96x96 residual blocks' shape
        (O._c(80, 32, 3, 1, 1), 2, (16, 16)),            # output block: Cin 80 = 64 + 16
        (O._t(160, 64, 3, 2, 1, 1), 2, (8, 8)),          # last transposed conv: two M tiles, the second 32 channels wide
        (O._c(384, 384, 3, 1, 1, True), 2, (6, 6)),      # three N tiles of 128, three M tiles
        (O._c(256, 256, 3, 1, 1, True), 2, (6, 6)),      # N tile 256
        (O._t(1024, 512, 3, 1, 0), 4, (1, 1)),           # 1x1 -> 3x3 transposed conv (GEMM form in the forward)
        (O._c(512, 512, 1, 1, 0), 4, (1, 1)),            # 1x1 conv on a 1x1 map: K = batch only
        (O._c(32, 64, 3, (3, 1), 1), 2, (20, 16)),       # audio encoder's (3,1) stride
        (O._n(32, 64, 5, (1, 2), 2), 2, (12, 24)),       # discriminator, k5 s(1,2), LeakyReLU, real bias gradient
    ]
    return out


def _id(c):
    r, n, hw = c
    return f"{r[0]}-{r[1]}to{r[2]}-k{r[3]}-s{r[4]}-p{r[5]}-op{r[6]}-res{int(r[7])}-n{n}-{hw[0]}x{hw[1]}"


@pytest.fixture(scope="module")
def ctx():
    from wav2lip_b200 import _lib
    return _lib.Context(0, _lib.PREC_BF16)


@pytest.mark.parametrize("case", _cases(), ids=_id)
def test_block_train_forward_backward(case, ctx):
    from wav2lip_b200 import _lib
    row, n, (H, W) = case
    kind, cin, cout, k, s, p, op, res = row
    (kh, kw), (sh, sw), (ph, pw) = O._pair(k), O._pair(s), O._pair(p)
    if kind != "t" and (H + 2 * ph < kh or W + 2 * pw < kw):
        pytest.skip("input smaller than the filter")
    g = torch.Generator().manual_seed((cin * 131 + cout * 17 + kh * 7 + kw * 3 + sh * 5 + sw + H * 11 + W + ord(kind)) % 100000)
    x = torch.randn((n, cin, H, W), generator=g)
    wshape = (cin, cout, kh, kw) if kind == "t" else (cout, cin, kh, kw)
    fan = cin * kh * kw
    w = torch.randn(wshape, generator=g) / fan ** 0.5
    b = 0.1 * torch.randn(cout, generator=g)
    gamma = 1 + 0.2 * torch.randn(cout, generator=g)
    beta = 0.1 * torch.randn(cout, generator=g)
    rmean, rvar = 0.1 * torch.randn(cout, generator=g), 0.5 + torch.rand(cout, generator=g)
    y_ref, saved = R.block_forward_train(x.double(), w.double(), b.double(), gamma.double(), beta.double(), row)
    dy = torch.randn(y_ref.shape, generator=g)
    ref = R.block_backward(dy.double(), x.double(), w.double(), gamma.double(), row, saved)     # exact operands
    same = reference_same_rounding(x, w, b, gamma, beta, dy, row)                                   # the kernels' rounding points

    li = _lib.LayerInfo()
    li.name = b"block"
    li.kind = {"c": _lib.BLOCK_CONV_BN_RELU, "t": _lib.BLOCK_CONVT_BN_RELU, "n": _lib.BLOCK_CONV_LRELU}[kind]
    li.cin, li.cout, li.kh, li.kw, li.sh, li.sw, li.ph, li.pw = cin, cout, kh, kw, sh, sw, ph, pw
    li.out_pad, li.residual = op, int(res)
    dev = "cuda:0"
    t = lambda a: a.float().contiguous().to(dev)
    xd, wd, bd, gd, bed, rmd, rvd, dyd = map(t, (x, w, b, gamma, beta, rmean, rvar, dy))
    yd = torch.empty(y_ref.shape, device=dev)
    dxd, dwd = torch.empty_like(xd), torch.full_like(wd, float("nan"))
    dbd, dgd, dbed = (torch.full((cout,), float("nan"), device=dev) for _ in range(3))
    P = lambda a: C.c_void_p(a.data_ptr())
    bn = kind != "n"
    _lib.check(ctx.lib.w2l_conv_block_train(ctx.h, C.byref(li), P(xd), n, H, W, P(wd), P(bd), P(gd) if bn else None,
                                            P(bed) if bn else None, P(rmd) if bn else None, P(rvd) if bn else None, P(dyd), P(yd),
                                            P(dxd), P(dwd), P(dbd), P(dgd) if bn else None, P(dbed) if bn else None, None))
    torch.cuda.synchronize()
    errs = {"y": rel_l2(yd.cpu(), same["y"]), "dx": rel_l2(dxd.cpu(), same["dx"]), "dw": rel_l2(dwd.cpu(), same["dw"])}
    loose = {"y": rel_l2(yd.cpu(), y_ref), "dx": rel_l2(dxd.cpu(), ref["dx"]), "dw": rel_l2(dwd.cpu(), ref["dw"])}
    if bn:
        errs["dgamma"] = rel_l2(dgd.cpu(), same["dgamma"])
        errs["dbeta"] = rel_l2(dbed.cpu(), same["dbeta"])
        errs["dbias_abs"] = dbd.abs().max().item()    # conv bias under a BatchNorm: exactly zero gradient
        # running averages as nn.BatchNorm2d updates them (momentum 0.1, unbiased variance, conv bias included in the mean)
        m = same["y"].numel() / cout
        m_ref = 0.9 * rmean.double() + 0.1 * (same["zmean"] + b.double())
        v_ref = 0.9 * rvar.double() + 0.1 * same["zvar"] * m / (m - 1)
        errs["rmean"] = rel_l2(rmd.cpu(), m_ref)
        errs["rvar"] = rel_l2(rvd.cpu(), v_ref)
    else:
        errs["db"] = rel_l2(dbd.cpu(), same["db"])
        loose["db"] = rel_l2(dbd.cpu(), ref["db"])
    bad = {k: v for k, v in errs.items() if not (v <= REL)}
    bad.update({"loose_" + k: v for k, v in loose.items() if not (v <= LOOSE)})
    assert not bad, ({k: float(f"{v:.3g}") for k, v in errs.items()}, {k: float(f"{v:.3g}") for k, v in loose.items()})


def test_block_train_rejects_bad_arguments(ctx):
    """The block descriptions w2l_conv_block_forward refuses, refused by the training entry too, with nothing launched."""
    from wav2lip_b200 import _lib
    from test_gpu_blocks import bad_layer_calls
    P = lambda a: C.c_void_p(a.data_ptr())
    for what, li, t in bad_layer_calls():
        dx, dw, grads = torch.empty_like(t["x"]), torch.empty_like(t["w"]), [torch.empty_like(t["b"]) for _ in range(3)]
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        with pytest.raises(_lib.W2LError):
            _lib.check(ctx.lib.w2l_conv_block_train(ctx.h, C.byref(li), P(t["x"]), 1, 8, 8, P(t["w"]), P(t["b"]), P(t["gamma"]),
                                                    P(t["beta"]), P(t["mean"]), P(t["var"]), P(t["y"]), P(t["y"]), P(dx),
                                                    P(dw), *map(P, grads), None))
        assert ctx.launch_count() == n0, what
