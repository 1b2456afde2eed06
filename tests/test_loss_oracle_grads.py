"""The float64 statements of the training tail in oracle/loss_oracle.py (generator head, embedding normalisation,
discriminator head, cosine / BCE / L1 loss gradients) against the installed torch, on the CPU:
  * at unclamped points, against torch.autograd in float64 through torch.sigmoid, F.normalize, F.cosine_similarity,
    F.binary_cross_entropy and F.l1_loss, to 1e-12 relative;
  * at every clamp (p in {0, 1, 2^-149, 1 - 2^-24}, a cosine of exactly 1, all-zero rows), against torch's own fp32
    forward and backward: the oracle evaluated on the same fp32 values must give torch's fp32 result to fp32 rounding.
tests/test_gpu_train_tail.py holds the CUDA kernels to these functions."""
import pytest
import torch
import torch.nn.functional as F

from oracle import loss_oracle as L

U24 = 2.0 ** -24


def close(got, ref, rel=1e-12):
    got, ref = torch.as_tensor(got).double(), torch.as_tensor(ref).double()
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs().max().item() if ref.numel() else 0.0
    scale = ref.abs().max().item() if ref.numel() else 0.0
    assert err <= rel * scale + 1e-300, f"max err {err:.3g}, scale {scale:.3g}"


def leaf(*shape, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale + offset).requires_grad_()


# ---- unclamped points: float64 autograd ----------------------------------------------------------------------------
@pytest.mark.parametrize("B,T", [(5, 0), (3, 5), (2, 5)])
def test_head_against_autograd(B, T):
    N, H, W = (T or 1) * B, 4, 3
    y32 = leaf(N, 32, H, W, seed=1)
    w, b = leaf(3, 32, seed=2, scale=0.2), leaf(3, seed=3)
    s = F.conv2d(y32, w.view(3, 32, 1, 1), b)
    if T:   # n = t*B + b -> (B, 3, T, H, W)
        s = s.view(T, B, 3, H, W).permute(1, 2, 0, 3, 4)
    g = torch.sigmoid(s)
    dg = torch.randn(g.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    ref = torch.autograd.grad(g, [y32, w, b], dg)
    got_g, got_s = L.head_forward(y32.detach(), w.detach(), b.detach(), B, T)
    close(got_g, g.detach())
    close(got_s, s.detach())
    dy32, dw, db, mw, mb = L.head_backward(y32.detach(), w.detach(), got_g, dg, B, T)
    close(dy32, ref[0])
    close(dw, ref[1])
    close(db, ref[2])
    assert (mw >= dw.abs()).all() and (mb >= db.abs()).all()


def test_head_layout_is_t_major():
    """swapping b and t in the unflatten changes the answer at B = 3, T = 5 (so the GPU test can tell them apart)"""
    B, T = 3, 5
    y32 = torch.arange(T * B, dtype=torch.float64).view(-1, 1, 1, 1).expand(-1, 32, 1, 1)
    g, s = L.head_forward(y32, torch.ones(3, 32), torch.zeros(3), B, T)
    for b in range(B):
        for t in range(T):
            assert s[b, 0, t, 0, 0].item() == 32.0 * (t * B + b)


def test_l2norm_against_autograd():
    r = leaf(6, 512, seed=5)
    de = torch.randn(6, 512, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    e = F.normalize(r, dim=1)
    close(L.l2norm(r.detach()), e.detach())
    close(L.l2norm_backward(r.detach(), de), torch.autograd.grad(e, r, de)[0])


@pytest.mark.parametrize("labels", ["mixed", "ones"])
@pytest.mark.parametrize("scale", [1.0, 0.03])
def test_cosine_bce_against_autograd(labels, scale):
    B = 6
    a, v = leaf(B, 512, seed=7, offset=0.3), leaf(B, 512, seed=8, offset=0.3)   # cosines well inside (0, 1)
    y = torch.tensor([[1.0], [0.0], [0.0], [1.0], [1.0], [0.0]], dtype=torch.float64) if labels == "mixed" else None
    d = F.cosine_similarity(a, v)
    loss = scale * F.binary_cross_entropy(d.unsqueeze(1), y if y is not None else torch.ones(B, 1, dtype=torch.float64))
    da_ref, dv_ref = torch.autograd.grad(loss, [a, v])
    got, da, dv, dd = L.cosine_bce_grad(a.detach(), v.detach(), y, scale)
    close(dd, d.detach())
    close(got, loss.detach())
    close(da, da_ref)
    close(dv, dv_ref)


@pytest.mark.parametrize("weight", [1.0, 0.07])
def test_bce_grad_against_autograd(weight):
    p = torch.rand(40, generator=torch.Generator().manual_seed(9), dtype=torch.float64).mul(0.98).add(0.01).requires_grad_()
    t = (torch.arange(40) % 3 == 0).double()
    loss = weight * F.binary_cross_entropy(p, t)
    close(L.bce(p.detach(), t) * weight, loss.detach())
    close(L.bce_grad(p.detach(), t, weight), torch.autograd.grad(loss, p)[0])


def test_disc_head_and_bce_against_autograd():
    N = 15
    feat, w, b = leaf(N, 512, seed=10), leaf(512, seed=11, scale=0.05), leaf(1, seed=12)
    p = torch.sigmoid(feat @ w + b)
    dp = torch.randn(N, generator=torch.Generator().manual_seed(13), dtype=torch.float64)
    ref = torch.autograd.grad(p, [feat, w, b], dp)
    got_p, _ = L.disc_head(feat.detach(), w.detach(), b.detach())
    close(got_p, p.detach())
    for got, r in zip(L.disc_head_backward(feat.detach(), w.detach(), got_p, dp), ref):
        close(got, r)
    # the hq step's three BCE means and their gradients
    pf = p.detach().clone().requires_grad_()
    pr = torch.rand(N, generator=torch.Generator().manual_seed(14), dtype=torch.float64).requires_grad_()
    losses, d_perc, d_fake, d_real = L.disc_bce(pf.detach(), pr.detach(), 0.07)
    for got, fn, x, w_ in ((losses[0], lambda q: F.binary_cross_entropy(q, torch.ones_like(q)), pf, 0.07),
                           (losses[1], lambda q: F.binary_cross_entropy(q, torch.ones_like(q)), pr, 1.0),
                           (losses[2], lambda q: F.binary_cross_entropy(q, torch.zeros_like(q)), pf, 1.0)):
        val = fn(x)
        close(got, val.detach())
    close(d_perc, torch.autograd.grad(0.07 * F.binary_cross_entropy(pf, torch.ones_like(pf)), pf)[0])
    close(d_fake, torch.autograd.grad(F.binary_cross_entropy(pf, torch.zeros_like(pf)), pf)[0])
    close(d_real, torch.autograd.grad(F.binary_cross_entropy(pr, torch.ones_like(pr)), pr)[0])
    assert L.disc_bce(pf.detach(), pr.detach(), 0.0)[0][0].item() == 0.0


def test_gen_loss_grad_against_autograd():
    """l1_scale sign(g - gt) + the expert's input gradient at channel 3t + c + the discriminator's at n = t*B + b, as
    autograd forms dL/dg of  w_l1 * L1(g, gt) + <dsync, stack_lower_halves(g)> + <ddisc, frames(g)>"""
    B, T, H, W = 3, 5, 8, 6
    gen = torch.Generator().manual_seed(15)
    g = torch.rand((B, 3, T, H, W), generator=gen, dtype=torch.float64).requires_grad_()
    gt = torch.rand((B, 3, T, H, W), generator=gen, dtype=torch.float64)
    gt[..., 0, 0] = g.detach()[..., 0, 0]   # ties: sign 0, as torch's L1 backward gives
    dsync = torch.randn((B, 3 * T, H // 2, W), generator=gen, dtype=torch.float64)
    ddisc = torch.randn((T * B, 3, H // 2, W), generator=gen, dtype=torch.float64)
    w_l1 = 0.9
    half = g[:, :, :, H // 2:]
    stacked = torch.cat([half[:, :, t] for t in range(T)], dim=1)                 # wav2lip_train.py's get_sync_loss input
    frames = torch.cat([half[:, :, t] for t in range(T)], dim=0)                 # Wav2Lip_disc_qual.to_2d: n = t*B + b
    loss = w_l1 * F.l1_loss(g, gt) + (dsync * stacked).sum() + (ddisc * frames).sum()
    ref = torch.autograd.grad(loss, g)[0]
    got = L.gen_loss_grad(g.detach(), gt, w_l1 / g.numel(), dsync, ddisc)
    close(got, ref)
    assert (got[..., 0, 0] == 0).all()


def test_combine_losses():
    assert L.combine_losses(2.0, 3.0, 5.0, 0.03, 0.07).item() == pytest.approx(0.03 * 2 + 0.07 * 5 + 0.9 * 3, rel=1e-15)


# ---- clamps: torch's fp32 forward and backward ---------------------------------------------------------------------
P_CLAMP = [0.0, 1.0, 2.0 ** -149, 1.0 - U24]


@pytest.mark.parametrize("t", [0.0, 1.0])
@pytest.mark.parametrize("p", P_CLAMP, ids=["0", "1", "2^-149", "1-2^-24"])
def test_bce_at_its_clamps_is_torchs(p, t):
    pt = torch.tensor([p], dtype=torch.float32, requires_grad=True)
    loss = F.binary_cross_entropy(pt, torch.tensor([t]))
    grad = torch.autograd.grad(loss, pt)[0]
    ref_l, ref_g = L.bce(pt.detach(), torch.tensor([t])), L.bce_grad(pt.detach(), torch.tensor([t]))
    assert torch.isfinite(ref_l) and torch.isfinite(ref_g).all()
    # torch's fp32 arithmetic rounds each step once: a few fp32 ulps (2^-149 * 1e12 is a denormal-scale product)
    assert abs(loss.item() - ref_l.item()) <= 4 * U24 * abs(ref_l.item()) + 2.0 ** -149, (loss.item(), ref_l.item())
    assert abs(grad.item() - ref_g.item()) <= 4 * U24 * abs(ref_g.item()) + 2.0 ** -149, (grad.item(), ref_g.item())


def test_bce_clamp_values():
    """the exact values the GPU test's saturated cases rely on"""
    assert L.bce(torch.tensor([1.0]), torch.tensor([0.0])).item() == 100.0          # fake term at p = 1
    assert L.bce(torch.tensor([0.0]), torch.tensor([1.0])).item() == 100.0
    assert L.bce_grad(torch.tensor([1.0]), torch.tensor([0.0])).item() == 1e12      # 1 / 1e-12 / n, n = 1
    assert L.bce_grad(torch.tensor([0.0, 0.0]), torch.tensor([1.0, 1.0]))[0].item() == -1e12 / 2


@pytest.mark.parametrize("case", ["a == v", "zero a", "zero a and v"])
@pytest.mark.parametrize("labels", ["ones", "zeros"])
def test_cosine_bce_at_its_clamps_is_torchs(case, labels):
    """d == 1 (to fp32 rounding) and zero rows: torch's fp32 cosine_loss forward and backward, fed the same fp32 values"""
    B, D = 4, 512
    gen = torch.Generator().manual_seed(16)
    v = torch.full((B, D), 0.5) if case == "a == v" else torch.randn((B, D), generator=gen)
    a = v.clone() if case == "a == v" else torch.zeros((B, D))
    if case == "zero a and v":
        v = torch.zeros((B, D))
    y = torch.ones(B, 1) if labels == "ones" else torch.zeros(B, 1)
    a32, v32 = a.clone().requires_grad_(), v.clone().requires_grad_()
    d32 = F.cosine_similarity(a32, v32)
    loss = F.binary_cross_entropy(d32.unsqueeze(1), y)
    da32, dv32 = torch.autograd.grad(loss, [a32, v32])
    # the oracle on torch's own fp32 cosine (a == v: torch gives 1 - 2^-24, not 1) reproduces torch's loss and dL/dd
    d = d32.detach().double()
    close(L.bce(d, y.reshape(-1)), loss.detach(), 4 * U24)
    _, da, dv, dd = L.cosine_bce_grad(a, v, y)
    assert torch.isfinite(da).all() and torch.isfinite(dv).all()
    if case == "a == v":
        assert dd.eq(1.0).all() and d.lt(1.0).all()       # float64 says 1 exactly; torch's fp32 lands one ulp below
        # the gradient of a cosine of 1 vanishes in float64; torch's is rounding noise: |dL/dd| times a few fp32 ulps
        # of the unit vector's 1/|a|
        assert da.abs().max().item() == 0.0 and dv.abs().max().item() == 0.0
        dldd32 = ((d32.detach() - y.reshape(-1)) / (d32.detach() * (1 - d32.detach())).clamp_min(1e-12) / B).abs()
        noise = dldd32 * 16 * U24 / a.norm(dim=1)
        assert (da32.abs().amax(1) <= noise).all() and (dv32.abs().amax(1) <= noise).all()
    else:
        close(da, da32, 8 * U24)
        close(dv, dv32, 8 * U24)


def test_normalize_zero_row_is_torchs():
    r = torch.zeros(2, 512).requires_grad_()
    r.data[1].normal_(generator=torch.Generator().manual_seed(17))
    e = F.normalize(r, dim=1)
    de = torch.randn(2, 512, generator=torch.Generator().manual_seed(18))
    g32 = torch.autograd.grad(e, r, de)[0]
    close(L.l2norm(r.detach()), e.detach(), 2 * U24)
    got = L.l2norm_backward(r.detach(), de)
    assert torch.equal(got[0], de[0].double() * 1e12)   # the clamp branch: de / 1e-12, no projection
    close(got[0], g32[0], 2 * U24)
    close(got[1], g32[1], 16 * U24)
