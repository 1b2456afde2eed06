"""The training tail against float64, from what each kernel itself read: the generator head (head_fwd / head_bwd /
head_bwd_finalize), the embedding normalisation (l2norm / l2norm_bwd), the discriminator head (disc_head /
disc_head_bwd), and the loss kernels that seed every backward (cosine_bce_bwd, gen_loss_grad, disc_bce,
combine_losses).  Their inputs come from the tapes (w2l_debug_train_tensor: exact 16-bit Y / DY / DX values, and the
fp32 copy of SyncNet's last-block outputs, TAPE_F32), the fp32 network outputs, w2l_train_last_output and the bound
weights and gradients, so the ~1e5 amplification of batch-statistics BatchNorm (DESIGN section 7) stays out, as in
tests/test_gpu_train_parity.py, whose helpers and bf16 bar (one rounding flip, ulp16) this file uses.  The float64
statements are oracle/loss_oracle.py's (pinned against torch on the CPU by tests/test_loss_oracle_grads.py).

Bars come from rounding analysis, per element (U = 2^-24):
  sigmoid (g, p)  the logit's fp32 fma chain, L U sum|terms| (L = 33 for the head's 32 taps + bias, 23 for the
                  discriminator's 16 per lane + 5 shuffles + bias), and __expf's documented 2 + floor(1.16 |x|) ulp,
                  pushed through fp32(1 / fp32(1 + e)) at both ends: both roundings are monotone, so the kernel's value
                  lies between the two fp32 results.  The bar is the larger distance from float64 to either end;
                  saturated logits (|s| > 17) give the exact fp32 value 1 and the bar collapses to float64's 1 - g.
  dy32, dfeat     one bf16 flip plus U times the fp32 roundings of dl = dg g (1 - g) and of the 3-term sum.
  dW, db          (per-thread chain + 16) U sum|dl f|: head_bwd's threads each sum ceil(M / (blocks * 256)) pixels,
                  then 5 shuffles, 8 warps, the fp64 block sum, one fp32 rounding and the accumulate add.
  loss-side       the cosine d (fp32 dots of 16 + 5 terms over the l2norm kernel's fp32 output) has a bound dd; dL/dd is
                  bounded over [d - dd, d + dd] (1025 points: the clamp 1e-12 makes it steep near 0 and 1), and the
                  normalisation backward maps the gradient's bound through (I - e e^T) / |r|.  BCE terms are monotone
                  in p, so the loss bars come from the interval's ends.
Every check prints a REPORT line with its largest err / bar."""
import math

import pytest
import torch

from oracle import loss_oracle as L
from oracle import w2l_oracle as O
from test_gpu_train_parity import (_CTX, ACCUMULATE, DISC, GEN, INPUT_GRAD, SYNC, WGRAD, Checker, NetRun, _ctx,
                                   _report, P)

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
F64 = torch.float64


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in _CTX.values():
        c.close()
    _CTX.clear()


def d64(t):
    return t.detach().to("cpu", F64)


def f32(t):
    """round float64 to fp32 (round to nearest even), kept in float64"""
    return t.float().double()


def sigmoid_f32_bounds(s, ds):
    """the interval of fp32(1 / fp32(1 + __expf(-s'))) over |s' - s| <= ds with __expf's documented error"""
    k = 2.0 + torch.floor(1.16 * (s.abs() + ds))
    e_lo = torch.exp(-(s + ds)) * (1.0 - k * 2.0 ** -23)
    e_hi = torch.exp(-(s - ds)) * (1.0 + k * 2.0 ** -23)
    den_lo, den_hi = f32(1.0 + e_lo), f32(1.0 + e_hi)
    return f32(1.0 / den_hi), f32(1.0 / den_lo)


def sigmoid_bar(s, ds):
    """bar of the kernel's fp32 sigmoid around float64 sigmoid(s): the larger distance to either end of the interval"""
    lo, hi = sigmoid_f32_bounds(s, ds)
    g = L.sigmoid64(s)
    return torch.maximum((hi - g).abs(), (g - lo).abs()) * (1 + 1e-12) + 1e-300, lo, hi


def sup_over(fn, lo, hi, mid, n=1025):
    """max |fn(x) - fn(mid)| and max |fn(x)| over x in [lo, hi] (per row), on n points and both ends"""
    t = torch.linspace(0.0, 1.0, n, dtype=F64)
    xs = lo.unsqueeze(-1) + (hi - lo).unsqueeze(-1) * t
    vals = fn(xs)
    ref = fn(mid.unsqueeze(-1))
    return (vals - ref).abs().amax(-1), vals.abs().amax(-1)


def block_index(ctx, net, name):
    for k, b in enumerate(ctx.train_blocks(net)):
        if b["name"] == name:
            return k
    raise AssertionError(f"no block {name}")


def tape(ctx, net, name, which):
    return ctx.train_tensor(net, block_index(ctx, net, name), which)


def report(what, chk):
    _report(what, chk.worst)


# ------------------------------------------------------------------------------------------------------------------
# the generator head
# ------------------------------------------------------------------------------------------------------------------
def head_fwd_check(chk, y32, w, b, g_got, B, T):
    g_ref, s = L.head_forward(y32, w, b, B, T)
    _, sm = L.head_forward(y32.abs(), w.abs(), b.abs(), B, T)   # sum |f w| + |b|, per element
    bar, lo, hi = sigmoid_bar(s, 33 * U * sm)
    chk.check("g", d64(g_got), g_ref, bar)
    torch_err = ((f32(torch.sigmoid(s.float()).double()) - g_ref).abs() / bar).max().item()
    return s, torch_err


def head_bwd_refs(y32, w, g_k, dg, B, T, dl_rel):
    """references and bars of dy32 (N,32,H,W), dW (3,32), db (3) from float64 dL/dg; dl_rel: relative error bound of the
    kernel's fp32 dl = dg g (1 - g) (its own roundings plus dg's)"""
    dy, dw, db, mw, mb = L.head_backward(y32, w, g_k, dg, B, T)
    dya, _, _, _, _ = L.head_backward(y32.abs(), w.abs(), g_k, dg.abs(), B, T)   # sum |dl| |w| (g (1 - g) >= 0)
    return dy, dw, db, (dl_rel + 3 * U) * dya + 1e-300, mw, mb


def head_case(B, T, bias, seed=0):
    ctx = _ctx()
    run = NetRun(ctx, GEN, B, 0, seed=seed)
    if T:
        mel, face = O.make_generator_inputs(B, seed=seed, t=T)
        run.T = T
        run.ins = [mel.cuda().contiguous(), face.cuda().contiguous()]
        run.outs = [torch.empty((B, 3, T, 96, 96), device="cuda"), None]
        gen = torch.Generator().manual_seed(200 + seed)
        run.dout = [torch.randn((B, 3, T, 96, 96), generator=gen).cuda(), None]
    if bias is not None:
        run.val["output_block.1.bias"].copy_(torch.tensor(bias, dtype=torch.float32))
    return ctx, run


HEAD_CASES = {   # id -> (B, T, head bias)
    "4d N=5": (5, 0, None),
    "5d B=3 T=5": (3, 5, None),
    "5d B=3 T=5 bias +-30": (3, 5, (30.0, -30.0, 30.0)),
    "4d N=5 bias -+30": (5, 0, (-30.0, 30.0, -30.0)),
}


@pytest.mark.parametrize("case", list(HEAD_CASES))
def test_head_through_the_bridge(case):
    """w2l_train_forward / w2l_train_backward of the generator: g from the output_block.0 Y tape and the bound head
    weights; dy32 (the output_block.0 DY tape), dW and db from dL/dg, then a second backward with W2L_TRAIN_ACCUMULATE
    adds the second dL/dg's gradients to the first's."""
    B, T, bias = HEAD_CASES[case]
    ctx, run = head_case(B, T, bias)
    chk = Checker(f"head {case}")
    run.forward(WGRAD)
    torch.cuda.synchronize()
    y32 = d64(tape(ctx, GEN, "output_block.0", 2))
    w, b = d64(run.val["output_block.1.weight"]).view(3, 32), d64(run.val["output_block.1.bias"])
    g_k = d64(run.outs[0])
    s, torch_err = head_fwd_check(chk, y32, w, b, run.outs[0], B, T)
    sat = (g_k == 1.0).sum().item(), (g_k < 1e-12).sum().item()
    M = y32.shape[0] * 9216
    nblk = torch.cuda.get_device_properties(0).multi_processor_count * 2
    chain = math.ceil(M / (nblk * 256)) + 16
    gen = torch.Generator().manual_seed(300)
    d2 = torch.randn(run.dout[0].shape, generator=gen).cuda()
    refs = []
    for i, (dg, flags) in enumerate(((run.dout[0], WGRAD), (d2, WGRAD | ACCUMULATE))):
        run.backward(flags, [dg, None])
        dy, dw, db, dybar, mw, mb = head_bwd_refs(y32, w, g_k, d64(dg), B, T, 3.1 * U)
        chk.check(f"dy32[{i}]", d64(tape(ctx, GEN, "output_block.0", 3)), dy, dybar, bf16_store=True)
        refs.append((dw, db, mw, mb))
        dw_ref, db_ref = sum(r[0] for r in refs), sum(r[1] for r in refs)
        # each pass's fp32 sum has its chain bar; the accumulate adds one rounding of the total
        bw = sum((chain + 4) * U * r[2] for r in refs) + U * dw_ref.abs() + 1e-300
        bb = sum((chain + 4) * U * r[3] for r in refs) + U * db_ref.abs() + 1e-300
        chk.check(f"dW[{i}]", d64(run.grad["output_block.1.weight"]).view(3, 32), dw_ref, bw)
        chk.check(f"db[{i}]", d64(run.grad["output_block.1.bias"]), db_ref, bb)
    print(f"REPORT head {case}: fp32 torch.sigmoid on the same s lands at {torch_err:.2f} of the g bar; "
          f"g == 1: {sat[0]}, g < 1e-12: {sat[1]}", flush=True)
    report(f"head {case}", chk)
    if bias is not None:
        assert sat[0] > 0 and sat[1] > 0


# ------------------------------------------------------------------------------------------------------------------
# SyncNet's embedding normalisation
# ------------------------------------------------------------------------------------------------------------------
LAST = {"audio": "audio_encoder.13", "face": "face_encoder.16"}
SYNC_WEIGHTS = ["random", "zero rows", "a == v"]


def sync_weights(val, which):
    """random: default init.  zero rows: the last blocks' BatchNorm gamma = 0, beta = -1 (every raw row is 0, the
    1e-12 / 1e-8 clamps are taken).  a == v: gamma = 0, beta = 0.5 on both encoders (a cosine of 1)."""
    if which == "random":
        return
    beta = -1.0 if which == "zero rows" else 0.5
    for name in LAST.values():
        val[f"{name}.conv_block.1.weight"].zero_()
        val[f"{name}.conv_block.1.bias"].fill_(beta)


def raw_rows(ctx, net):
    """the fp32 raw embeddings (audio, face) of the last plan of `net` (TAPE_F32), and a check that they are the Y tape"""
    out = []
    for name in (LAST["audio"], LAST["face"]):
        r = tape(ctx, net, name, 9)
        assert r is not None and r.shape[1:] == (512, 1, 1), name
        y = tape(ctx, net, name, 2)
        assert torch.equal(r.to(torch.bfloat16).float(), y), f"{name}: the fp32 copy is not the Y tape's source"
        out.append(d64(r).flatten(1))
    assert tape(ctx, net, "face_encoder.0", 9) is None   # a block without an fp32 output
    return out


def l2norm_fwd_bar(r):
    return 14 * U * L.l2norm(r).abs() + 1e-300


def l2norm_bwd_ref(r, de, dde=None):
    """float64 l2norm backward of de and its bar: the kernel's fp32 roundings (sums of 16 + 5 terms) plus, when de is
    itself the kernel's fp32 value known to within dde, that bound mapped through (I - e e^T) / |r|"""
    ref = L.l2norm_backward(r, de)
    n = r.norm(dim=1, keepdim=True)
    inv = 1.0 / n.clamp_min(L.NORM_EPS)
    on = (n > L.NORM_EPS).double()
    e = r * inv
    proj = on * (r * de).sum(1, keepdim=True) * inv * inv
    dproj = on * U * (21 * (r * de).abs().sum(1, keepdim=True) + 26 * (r * de).sum(1, keepdim=True).abs()) * inv * inv
    bar = (r.abs() * dproj + 2 * U * (de.abs() + (r * proj).abs())) * inv + 13 * U * ref.abs()
    if dde is not None:
        bar = bar + (dde + e.abs() * on * (e.abs() * dde).sum(1, keepdim=True)) * inv
    return ref, bar + 1e-300


@pytest.mark.parametrize("weights", SYNC_WEIGHTS)
def test_syncnet_normalisation_through_the_bridge(weights):
    """out0 / out1 against float64 normalize(F32 tape); the last audio and face blocks' DY tapes against float64
    l2norm backward of the bound output gradients (one bf16 flip)."""
    ctx = _ctx()
    run = NetRun(ctx, SYNC, 8, 0, seed=1)
    sync_weights(run.val, weights)
    chk = Checker(f"l2norm {weights}")
    run.forward(WGRAD | INPUT_GRAD)
    run.backward(WGRAD | INPUT_GRAD)
    ra, rf = raw_rows(ctx, SYNC)
    for i, (r, name) in enumerate(((ra, "audio"), (rf, "face"))):
        chk.check(f"out{i}", d64(run.outs[i]), L.l2norm(r), l2norm_fwd_bar(r))
        ref, bar = l2norm_bwd_ref(r, d64(run.dout[i]))
        chk.check(f"dy {name}", d64(tape(ctx, SYNC, LAST[name], 3)).flatten(1), ref, bar, bf16_store=True)
    if weights == "zero rows":
        assert ra.abs().max() == 0 and rf.abs().max() == 0
    if weights == "a == v":
        assert torch.equal(ra, rf)
    report(f"l2norm {weights}", chk)


# ------------------------------------------------------------------------------------------------------------------
# the sync loss inside the fused steps: cosine_bce_bwd and the loss
# ------------------------------------------------------------------------------------------------------------------
def check_sync_loss(chk, ctx, net, loss_got, y, scale):
    """the loss and both last blocks' DY tapes of the last plan of `net` in float64 from the F32 tapes and y"""
    ra, rf = raw_rows(ctx, net)
    a, v = L.l2norm(ra), L.l2norm(rf)
    B = a.shape[0]
    yv = torch.ones(B, dtype=F64) if y is None else d64(y).flatten()
    _, da, dv, d = L.cosine_bce_grad(a, v, yv, scale)
    loss = L.bce(d, yv)   # the step reports the unscaled sync loss
    # bound of the kernel's d: fp32 dots of 16 + 5 terms over inputs within 14 U, the norms' and the division's roundings
    na, nv, nn = L._cos_norms(a, v)
    dd = U * (51 * (a * v).abs().sum(1) / nn.squeeze(1) + 53 * d.abs())
    fn = lambda x: scale * (x - yv.view(-1, 1)) / (x * (1 - x)).clamp_min(L.BCE_DEN_MIN) / B
    df, fsup = sup_over(fn, d - dd, d + dd, d)
    df, fsup = (df + 5 * U * fsup).unsqueeze(1), fsup.unsqueeze(1)
    for name, x, z, nx, grad, r in (("audio", a, v, na, da, ra), ("face", v, a, nv, dv, rf)):
        beta = (z - d.unsqueeze(1) * x * ((nn / nx) / nx)) / nn   # dd/dx
        dde = df * beta.abs() + fsup * (U * (42 * z.abs() / nn + 44 * (d.unsqueeze(1) * x).abs() / (nx * nx))
                                        + dd.unsqueeze(1) * x.abs() / (nx * nx))
        ref, bar = l2norm_bwd_ref(r, grad, dde)
        chk.check(f"dy {name}", d64(tape(ctx, net, LAST[name], 3)).flatten(1), ref, bar, bf16_store=True)
    # the loss: BCE is monotone in d, so its bound comes from the interval's ends (clipped to [0, 1]: the kernel's
    # clamps give 1's values beyond it)
    ends = [L.bce_terms((d + s * dd).clamp(0, 1), yv) for s in (-1.0, 1.0)]
    terms = L.bce_terms(d, yv)
    lbar = (torch.maximum((ends[0] - terms).abs(), (ends[1] - terms).abs()).mean()
                    + 16 * U * terms.abs().mean() + dd.max())
    assert math.isfinite(loss_got), loss_got
    chk.check("loss", torch.tensor([loss_got], dtype=F64), loss.reshape(1), lbar.reshape(1) + 1e-300)
    return d


@pytest.mark.parametrize("weights", SYNC_WEIGHTS)
def test_syncnet_step_sync_loss(weights):
    """w2l_syncnet_train_step at B = 6, labels mixed 0 / 1: the loss and both encoders' DY tapes from the F32 tapes.
    zero rows: d = 0, so d (1 - d) clamps at 1e-12 (dL/dd = -1e12 / B for y = 1) and the loss is 100 per positive row;
    a == v: d is 1 to fp32 rounding."""
    from wav2lip_b200.models import SyncNet_color
    from wav2lip_b200.training import SyncNetTrainStep
    sd = O.make_state_dict("syncnet", 2, init="default")
    sync_weights(sd, weights)
    model = SyncNet_color()
    model.load_state_dict(sd, strict=True)
    model = model.cuda().train()
    mel, face = O.make_syncnet_inputs(6, seed=5)
    y = torch.tensor([[1.0], [0.0], [0.0], [1.0], [1.0], [0.0]]).cuda()
    step = SyncNetTrainStep(model, lr=1e-4)
    loss = step(face.cuda(), mel.cuda(), y).item()
    chk = Checker(f"syncnet step {weights}")
    d = check_sync_loss(chk, step.b.ctx, SYNC, loss, y, 1.0)
    if weights == "zero rows":
        assert loss == 50.0, loss   # three positive rows at d = 0: -max(log 0, -100) = 100 each, over B = 6
    print(f"REPORT syncnet step {weights}: d in [{d.min().item():.6g}, {d.max().item():.6g}], loss {loss:.6g}", flush=True)
    report(f"syncnet step {weights}", chk)


# ------------------------------------------------------------------------------------------------------------------
# the wav2lip step: sync loss scaled by syncnet_wt, gen_loss_grad through the head
# ------------------------------------------------------------------------------------------------------------------
def test_wav2lip_step_sync_loss_and_generator_gradient():
    """w2l_wav2lip_train_step at B = 3, T = 5, syncnet_wt = 0.03: the expert's loss and DY tapes (labels all ones, scale
    syncnet_wt); then dL/dg = l1_scale sign(g - gt) + the expert's first face block's DX tape at channel 3t + c of the
    lower half, pushed through the head's backward, against the output block's DY tape and the head's gradients.  A
    second, identical step takes gt = g on a mask of pixels, so sign(0) = 0 is exercised; determinism (tested elsewhere)
    makes its g the first step's, which is asserted."""
    from wav2lip_b200.training import Wav2LipTrainStep
    from test_gpu_train_steps import _nets, _train_inputs
    B, T, WS = 3, 5, 0.03
    x, indiv_mels, mel, gt = (t.cuda() for t in _train_inputs(B, seed=21))
    model, _, syncnet = _nets()
    before = {k: v.clone() for k, v in model.state_dict().items()}
    step = Wav2LipTrainStep(model, syncnet, lr=1e-4, syncnet_wt=WS)
    step(x, indiv_mels, mel, gt)
    g1 = step.last_output(B, T)
    with torch.no_grad():   # restore the pre-step weights and statistics in place (the binding keeps its pointers)
        for k, v in model.state_dict().items():
            v.copy_(before[k])
    model.mark_weights_dirty()
    mask = torch.rand(g1.shape, generator=torch.Generator().manual_seed(22)).cuda() < 0.25
    gt2 = torch.where(mask, g1, gt)
    losses = step(x, indiv_mels, mel, gt2).cpu()
    g_k = step.last_output(B, T)
    assert torch.equal(g_k, g1), "the repeated step's g differs from the first step's"
    ctx = step.b.ctx
    chk = Checker("wav2lip step")
    check_sync_loss(chk, ctx, SYNC, losses[0].item(), None, torch.tensor(WS, dtype=torch.float32).item())
    numel = g_k.numel()
    l1_scale = (torch.tensor(1.0, dtype=torch.float32) - torch.tensor(WS, dtype=torch.float32)) / float(numel)
    dsync = d64(tape(ctx, SYNC, "face_encoder.0", 6))
    assert dsync.shape == (B, 15, 48, 96)
    g64 = d64(g_k)
    dg = L.gen_loss_grad(g64, d64(gt2), float(l1_scale), dsync=dsync)
    assert (g64 == d64(gt2))[mask.cpu()].all() and (dg[..., :48, :][mask.cpu()[..., :48, :]] == 0).all()
    y32 = d64(tape(ctx, GEN, "output_block.0", 2))
    w = d64(before["output_block.1.weight"]).view(3, 32)
    dy, dw, db, dybar, mw, mb = head_bwd_refs(y32, w, g64, dg, B, T, 4.1 * U)   # dg's fp32 sum: one rounding more
    chk.check("dy32", d64(tape(ctx, GEN, "output_block.0", 3)), dy, dybar, bf16_store=True)
    M = y32.shape[0] * 9216
    nblk = torch.cuda.get_device_properties(0).multi_processor_count * 2
    chain = math.ceil(M / (nblk * 256)) + 16
    chk.check("dW", d64(step.b.grads["output_block.1.weight"]).view(3, 32), dw, (chain + 5) * U * mw + 1e-300)
    chk.check("db", d64(step.b.grads["output_block.1.bias"]), db, (chain + 5) * U * mb + 1e-300)
    lt = [losses[i].item() for i in range(4)]
    tot = L.combine_losses(lt[0], lt[1], lt[2], float(torch.tensor(WS, dtype=torch.float32)), 0.0)
    chk.check("total", torch.tensor([lt[3]], dtype=F64), tot.reshape(1),
              torch.tensor([4 * U * (abs(WS * lt[0]) + abs(lt[1])) + 1e-300], dtype=F64))
    report("wav2lip step", chk)


def test_disc_input_gradient_scatter_through_the_bridge():
    """w2l_train_backward(disc, ..., dinput) at B = 3, T = 5 is the first block's DX tape scattered to the lower half
    at n = t*B + b, bit for bit; the upper half is 0."""
    ctx = _ctx()
    B, T = 3, 5
    run = NetRun(ctx, DISC, B, T)
    out = run.step(WGRAD | INPUT_GRAD)
    dx = d64(tape(ctx, DISC, "face_encoder_blocks.0.0", 6))
    assert dx.shape == (T * B, 3, 48, 96)
    ref = torch.zeros((B, 3, T, 96, 96), dtype=F64)
    ref[..., 48:, :] = dx.view(T, B, 3, 48, 96).permute(1, 2, 0, 3, 4)
    assert torch.equal(d64(out["dinput"]), ref)
    assert torch.equal(L.gen_loss_grad(torch.zeros_like(ref), torch.zeros_like(ref), 0.0, ddisc=dx), ref)
    print("REPORT disc scatter: bit-identical", flush=True)


# ------------------------------------------------------------------------------------------------------------------
# the hq step: disc_bce, the discriminator head, combine_losses
# ------------------------------------------------------------------------------------------------------------------
HQ_CASES = {"bias 0": (0.0, 0.07), "bias +40": (40.0, 0.07), "bias -40": (-40.0, 0.07), "bias 0, disc_wt 0": (0.0, 0.0)}
LAST_DISC = "face_encoder_blocks.6.1"


def disc_probs(feat, w, b):
    p, s = L.disc_head(feat, w, b)
    _, sm = L.disc_head(feat.abs(), w.abs(), b.abs())
    bar, lo, hi = sigmoid_bar(s, 23 * U * sm)
    return p, lo, hi


def dl_of(grad_fn, p_lo, p_hi, p_mid):
    """dl = dBCE/dp * p (1 - p) (disc_head_bwd's logit gradient) over the kernel's p interval: value at float64 p, bound"""
    fn = lambda q: grad_fn(q) * q * (1 - q)
    dev, sup = sup_over(fn, p_lo, p_hi, p_mid, n=257)
    return fn(p_mid), dev + 8 * U * sup + 1e-300


@pytest.mark.parametrize("case", list(HQ_CASES))
def test_hq_step_disc_losses_and_head(case):
    """w2l_hq_wav2lip_train_step at B = 3, T = 5 (no sync term).  After the step the discriminator's last plan is the
    one on gt: p_real from its Y tape and the pre-step head weights, its DY tape against float64 d_real w.  p_fake: the
    pre-step discriminator weights are restored and w2l_train_forward(disc, g) reruns the step's g plan (same weights,
    same input, same plan: the values the step saw); its DY tape is still the step's fake pass.  Losses [2], [4], [5]
    against float64 BCE, [3] against the weighted sum of the step's own [0..2], and the accumulated binary_pred
    gradient (real + fake).  bias +40: p = 1 exactly in fp32, the fake term clamps at 100 and d_fake = 1e12 / n;
    bias -40: p ~ 4e-18, the perceptual and real terms are 40, unclamped, and the fake term is p itself."""
    from wav2lip_b200 import _lib
    from wav2lip_b200.training import HQWav2LipTrainStep
    from test_gpu_train_steps import _nets, _train_inputs
    bias, WD = HQ_CASES[case]
    B, T = 3, 5
    N = B * T
    x, indiv_mels, mel, gt = (t.cuda() for t in _train_inputs(B, seed=31))
    dsd = O.make_state_dict("disc", 3, init="default")
    dsd["binary_pred.0.bias"].fill_(bias)
    model, disc, _ = _nets(disc_sd=dsd)
    dbefore = {k: v.clone() for k, v in disc.state_dict().items()}
    step = HQWav2LipTrainStep(model, disc, None, disc_wt=WD)
    losses = step(x, indiv_mels, mel, gt).cpu().double()
    ctx = step.b.ctx
    g_k = step.last_output(B, T)
    w, b = d64(dbefore["binary_pred.0.weight"]).flatten(), d64(dbefore["binary_pred.0.bias"])
    chk = Checker(f"hq {case}")
    # the real pass: the plan on gt
    feat_r = d64(tape(ctx, DISC, LAST_DISC, 2)).flatten(1)
    dfeat_r = d64(tape(ctx, DISC, LAST_DISC, 3)).flatten(1)
    pr, pr_lo, pr_hi = disc_probs(feat_r, w, b)
    one = lambda q: torch.ones_like(q)
    dl_r, dl_r_bar = dl_of(lambda q: (q - 1) / (q * (1 - q)).clamp_min(L.BCE_DEN_MIN) / N, pr_lo, pr_hi, pr)
    chk.check("dfeat real", dfeat_r, dl_r.unsqueeze(1) * w, dl_r_bar.unsqueeze(1) * w.abs() + 1e-300, bf16_store=True)
    # the fake pass: rerun the g plan with the pre-step weights
    with torch.no_grad():
        for k, v in disc.state_dict().items():
            v.copy_(dbefore[k])
    p_fake = torch.empty((N, 1), device="cuda")
    _lib.check(ctx.lib.w2l_train_forward(ctx.h, DISC, P(g_k), None, P(p_fake), None, B, T, WGRAD | INPUT_GRAD, None))
    torch.cuda.synchronize()
    feat_f = d64(tape(ctx, DISC, LAST_DISC, 2)).flatten(1)
    dfeat_f = d64(tape(ctx, DISC, LAST_DISC, 3)).flatten(1)
    pf, pf_lo, pf_hi = disc_probs(feat_f, w, b)
    pbar = torch.maximum((pf_hi - pf).abs(), (pf - pf_lo).abs()) * (1 + 1e-12) + 1e-300
    chk.check("p_fake", d64(p_fake).flatten(), pf, pbar)
    dl_f, dl_f_bar = dl_of(lambda q: q / (q * (1 - q)).clamp_min(L.BCE_DEN_MIN) / N, pf_lo, pf_hi, pf)
    chk.check("dfeat fake", dfeat_f, dl_f.unsqueeze(1) * w, dl_f_bar.unsqueeze(1) * w.abs() + 1e-300, bf16_store=True)
    # the three BCE means: monotone in p, bars from the ends of the p intervals, plus the fp32 sums' roundings
    def bce_check(q, p, lo, hi, t, got):
        terms = L.bce_terms(p, t)
        ends = [L.bce_terms(e, t) for e in (lo, hi)]
        bar = torch.maximum((ends[0] - terms).abs(), (ends[1] - terms).abs()).mean() + 16 * U * terms.abs().mean()
        chk.check(q, got.reshape(1), terms.mean().reshape(1), bar.reshape(1) + 1e-300)
    bce_check("loss[4] real", pr, pr_lo, pr_hi, one(pr), losses[4])
    bce_check("loss[5] fake", pf, pf_lo, pf_hi, torch.zeros_like(pf), losses[5])
    if WD > 0:
        bce_check("loss[2] perceptual", pf, pf_lo, pf_hi, one(pf), losses[2])
    else:
        assert losses[2].item() == 0.0
    tot = L.combine_losses(losses[0], losses[1], losses[2], 0.0, float(torch.tensor(WD, dtype=torch.float32)))
    chk.check("loss[3] total", losses[3].reshape(1), tot.reshape(1),
              (4 * U * (WD * losses[2].abs() + losses[1].abs())).reshape(1) + 1e-300)
    # binary_pred's gradient: the real pass's, then the fake pass's accumulated onto it
    gw, gb = d64(step.db.grads["binary_pred.0.weight"]).flatten(), d64(step.db.grads["binary_pred.0.bias"])
    dw_ref = dl_r @ feat_r + dl_f @ feat_f
    mag = (dl_r.abs() + dl_r_bar) @ feat_r.abs() + (dl_f.abs() + dl_f_bar) @ feat_f.abs()
    chk.check("dw", gw, dw_ref, (N + 2) * U * mag + dl_r_bar @ feat_r.abs() + dl_f_bar @ feat_f.abs() + 1e-300)
    db_ref = dl_r.sum() + dl_f.sum()
    chk.check("db", gb, db_ref.reshape(1),
              ((N + 2) * U * (dl_r.abs().sum() + dl_f.abs().sum()) + dl_r_bar.sum() + dl_f_bar.sum()).reshape(1) + 1e-300)
    print(f"REPORT hq {case}: p_real in [{pr.min().item():.3g}, {pr.max().item():.3g}], p_fake in "
          f"[{pf.min().item():.3g}, {pf.max().item():.3g}], losses {[round(v, 6) for v in losses.tolist()]}", flush=True)
    if bias == 40.0:   # the clamp: 100 per row, then the fp32 mean's rounding
        assert (p_fake == 1.0).all() and abs(losses[5].item() - 100.0) <= 4 * U * 100.0
    if bias == -40.0:  # unclamped logs: -log(p) ~ 40 for the real and perceptual terms, the fake term p itself
        assert 30.0 < losses[4].item() < 50.0 and 0 < losses[5].item() < 1e-16
    report(f"hq {case}", chk)
