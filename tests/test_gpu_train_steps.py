"""The fused steps of hq_wav2lip_train.py:212-256 (`HQWav2LipTrainStep`, w2l_hq_wav2lip_train_step) and of
color_syncnet_train.py:149-163 (`SyncNetTrainStep`, w2l_syncnet_train_step), and the fused steps' Adam state in
torch.optim.Adam's format (w2l_adam_state): against the real scripts' steps (tests/golden/train.npz), the oracle, float64
autograd, the autograd bridge and torch's own Adam.  Bars follow tests/test_gpu_train_nets.py, whose docstring says why
they are what they are (bf16 operands under batch-statistics BatchNorm)."""
import copy
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import w2l_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel_l2(got, ref):
    return ((got.double().cpu() - ref.double().cpu()).norm() / (ref.double().cpu().norm() + 1e-30)).item()


def fp3(t):
    f = t.detach().double().flatten().cpu()
    return np.array([f.sum().item(), f.abs().sum().item(), f.abs().max().item()])


def relu_active(sd, beta=3.0):
    return {k: (torch.full_like(v, beta) if k.endswith("conv_block.1.bias") else v.clone()) for k, v in sd.items()}


def report(name, rep):
    import json
    print("REPORT " + json.dumps({"test": name, **rep}, default=str), flush=True)


def summarize(errs):
    v = sorted(errs.values())
    worst = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    return {"n": len(v), "median": round(v[len(v) // 2], 4), "p90": round(v[int(len(v) * 0.9)], 4), "max": round(v[-1], 4),
            "worst": [(k, round(e, 4)) for k, e in worst]}


def _train_inputs(B, seed, T=5):
    g = torch.Generator().manual_seed(seed)
    indiv_mels, x = O.make_generator_inputs(B, seed=seed, t=T)
    mel = torch.rand((B, 1, 80, 16), generator=g) * 8 - 4
    gt = torch.rand((B, 3, T, 96, 96), generator=g)
    return x, indiv_mels, mel, gt


def _nets(gen_seed=0, disc_seed=3, sync_seed=1, gen_sd=None, disc_sd=None, sync_sd=None):
    from wav2lip_b200.models import SyncNet_color, Wav2Lip, Wav2Lip_disc_qual
    model, disc, syncnet = Wav2Lip(), Wav2Lip_disc_qual(), SyncNet_color()
    model.load_state_dict(gen_sd if gen_sd is not None else O.make_state_dict("generator", gen_seed, init="default"), strict=True)
    disc.load_state_dict(disc_sd if disc_sd is not None else O.make_state_dict("disc", disc_seed, init="default"), strict=True)
    syncnet.load_state_dict(sync_sd if sync_sd is not None else O.make_state_dict("syncnet", sync_seed, init="default"), strict=True)
    return model.cuda().train(), disc.cuda().train(), syncnet.cuda().train()


def _syncnet(sd):
    from wav2lip_b200.models import SyncNet_color
    s = SyncNet_color()
    s.load_state_dict(sd, strict=True)
    return s.cuda().train()


def _sd_rel(module, ref_fp):
    got = np.stack([fp3(v) for v in module.state_dict().values()])
    return np.abs(got[:, 1] - ref_fp[:, 1]) / np.maximum(ref_fp[:, 1], 1e-12)


# ----------------------------------------------------------------------------------------------------------------------
# hq_wav2lip_train.py
# ----------------------------------------------------------------------------------------------------------------------
def test_hq_fused_step_against_the_reference_golden(golden_dir):
    """Two iterations of hq_wav2lip_train.py:212-256 as native calls against the REAL script's step (train.npz hq0/hq1),
    with the bars the autograd-bridge version of this test uses."""
    from wav2lip_b200.training import HQWav2LipTrainStep
    gold = np.load(os.path.join(golden_dir, "train.npz"))
    model, disc, syncnet = _nets()
    expert0 = {k: v.clone() for k, v in syncnet.state_dict().items()}
    step = HQWav2LipTrainStep(model, disc, syncnet, lr=1e-4, disc_lr=1e-4, syncnet_wt=0.03, disc_wt=0.07)
    x, indiv_mels, mel, gt = (t.cuda() for t in _train_inputs(2, seed=8))
    for it in range(2):
        lo = step(x, indiv_mels, mel, gt).cpu().numpy()              # [sync, l1, perceptual, loss, real, fake]
        got = np.array([lo[3], lo[0], lo[2], lo[1], lo[4], lo[5]])  # the golden's order: loss, sync, perceptual, l1, real, fake
        ref = gold[f"hq{it}_losses"]
        rel = np.abs(got - ref) / np.abs(ref)
        dnames = list(gold[f"hq{it}_disc_grad_names"])
        assert dnames == list(step.db.grads.keys())
        dfp = np.stack([fp3(step.db.grads[n]) for n in dnames])
        drel = np.abs(dfp[:, 1] - gold[f"hq{it}_disc_grad_fp"][:, 1]) / np.maximum(gold[f"hq{it}_disc_grad_fp"][:, 1], 1e-12)
        gnames = list(model.state_dict().keys())
        is_stat = np.array([("running" in n) or ("num_batches" in n) for n in gnames])
        grel = _sd_rel(model, gold[f"hq{it}_gen_sd_fp"])
        dsrel = _sd_rel(disc, gold[f"hq{it}_disc_sd_fp"])
        report(f"hq_fused_step{it}", {"losses": got.tolist(), "ref": ref.tolist(), "loss_rel": rel.tolist(),
                                      "disc_grad_fp_rel_max": float(drel.max()), "disc_grad_fp_rel_median": float(np.median(drel)),
                                      "gen_sd_rel_max": float(grel[~is_stat].max()), "gen_stat_rel_max": float(grel[is_stat].max()),
                                      "disc_sd_rel_max": float(dsrel.max())})
        assert abs(lo[3] - (0.03 * lo[0] + 0.07 * lo[2] + 0.90 * lo[1])) <= 1e-6, lo   # the weighted sum itself
        assert rel[3] <= 2e-3, (it, got, ref)                                        # L1
        # sync: the expert's BatchNorms see B = 2 samples (zhat = +-1), so bf16 moves this loss by several per cent
        # (measured 0.097 at step 0, 0.038 at step 1)
        assert rel[1] <= 0.12, (it, got, ref)
        assert rel[2] <= 2e-2 and rel[4] <= 2e-2 and rel[5] <= 2e-2, (it, got, ref)  # the three BCE terms
        assert rel[0] <= 1e-2, (it, got, ref)
        assert np.median(drel) <= 0.1 and drel.max() <= 0.5, (it, drel)
        assert grel[~is_stat].max() <= 6e-3 and dsrel.max() <= 6e-3, (it, grel[~is_stat].max(), dsrel.max())
        assert grel[is_stat].max() <= 6e-2, (it, grel[is_stat].max())
        # the expert ran in train mode (the script never .eval()s it): buffers moved, weights did not
        now = syncnet.state_dict()
        for k, v in expert0.items():
            if "running" in k:
                assert not torch.equal(now[k], v), k
            elif not k.endswith("num_batches_tracked"):
                assert torch.equal(now[k], v), k
            else:
                assert int(now[k]) == it + 1, k


def _disc_grad_errors_f64(disc_sd, fake, real, got):
    """float64 autograd of BCE(disc(real), 1) + BCE(disc(fake), 0) on the oracle (hq_wav2lip_train.py:247-253) -> relative
    L2 error of every discriminator gradient in `got`."""
    leaves = {k: v.double().clone().requires_grad_(True) for k, v in disc_sd.items() if v.dtype.is_floating_point}
    pr = O.disc_forward(leaves, real.double().cpu())
    pf = O.disc_forward(leaves, fake.double().cpu())
    loss = F.binary_cross_entropy(pr, torch.ones_like(pr)) + F.binary_cross_entropy(pf, torch.zeros_like(pf))
    names = list(leaves)
    ref = dict(zip(names, torch.autograd.grad(loss, [leaves[k] for k in names])))
    return {n: rel_l2(got[n], ref[n]) for n in names}


@pytest.mark.parametrize("disc_wt", [0.07, 0.0])
def test_hq_fused_step_at_the_scripts_starting_weights_against_the_oracle(disc_wt):
    """syncnet_wt = 0 (hq_wav2lip_train.py starts that way): losses against oracle.train_oracle.hq_train_step; the
    discriminator's gradients against float64 autograd on the step's own g.  disc_wt = 0: no perceptual term, the
    discriminator still trains, and the generator's gradient is exactly the L1-only step's (Wav2LipTrainStep)."""
    from oracle import train_oracle as TO
    from wav2lip_b200.training import HQWav2LipTrainStep, Wav2LipTrainStep
    gen_sd = O.make_state_dict("generator", 0, init="default")
    disc_sd = O.make_state_dict("disc", 3, init="default")
    x, indiv_mels, mel, gt = _train_inputs(2, seed=9)
    r = TO.hq_train_step({k: v.clone() for k, v in gen_sd.items()}, {k: v.clone() for k, v in disc_sd.items()}, {},
                         x, indiv_mels, mel, gt, syncnet_wt=0.0, disc_wt=disc_wt)
    model, disc, _ = _nets(gen_sd=gen_sd, disc_sd=disc_sd)
    step = HQWav2LipTrainStep(model, disc, None, syncnet_wt=0.0, disc_wt=disc_wt)
    lo = step(x.cuda(), indiv_mels.cuda(), mel.cuda(), gt.cuda()).cpu().numpy()
    g = step.last_output()
    errs = _disc_grad_errors_f64(disc_sd, g, gt, step.db.grads)
    rep = summarize(errs)
    rep.update({"losses": lo.tolist(), "ref": [float(r[k]) for k in ("sync_loss", "l1", "perceptual", "loss", "disc_real", "disc_fake")]})
    report(f"hq_fused_oracle_wt{disc_wt}", rep)
    assert lo[0] == 0.0
    assert abs(lo[1] - float(r["l1"])) <= 2e-3 * float(r["l1"]), rep
    for i, k in ((4, "disc_real"), (5, "disc_fake")):
        assert abs(lo[i] - float(r[k])) <= 2e-2 * float(r[k]), (k, rep)
    assert rep["median"] <= 0.25 and rep["max"] <= 0.35, rep
    moved = [n for n, p in disc.named_parameters() if not torch.equal(p.detach().cpu(), disc_sd[n])]
    assert len(moved) == len(list(disc.parameters())), "every discriminator tensor takes an Adam step"
    if disc_wt > 0:
        assert abs(lo[2] - float(r["perceptual"])) <= 2e-2 * float(r["perceptual"]), rep
        assert abs(lo[3] - (disc_wt * lo[2] + (1 - disc_wt) * lo[1])) <= 1e-6, lo
    else:
        assert lo[2] == 0.0 and lo[3] == lo[1], lo
        m2, _, _ = _nets(gen_sd=gen_sd)
        ref_step = Wav2LipTrainStep(m2, None, syncnet_wt=0.0)
        ref_step(x.cuda(), indiv_mels.cuda(), mel.cuda(), gt.cuda())
        assert torch.equal(ref_step.b.arena, step.b.arena), "generator gradient of the hq step without the perceptual term"


@pytest.mark.parametrize("ws", [0.0, 0.03])
def test_hq_fused_step_equals_the_bridge(ws):
    """B = 8, T = 5, step 0, disc_wt 0.07: the fused step against hq_wav2lip_train.py's statements on the mirrors (the
    autograd bridge), which build the same plans and run the same kernels.
      * g is bit-identical; the six losses agree to the loss arithmetic's rounding; losses[5] — from the g tape the step
        reuses — equals BCE(disc(g), 0) recomputed on the step's own g;
      * every discriminator gradient (real + fake) is bit-identical: its inputs are g and gt, and the BCE gradients follow
        torch's operation order;
      * without the sync term every generator gradient is bit-identical too: dL/dg = L1 + perceptual input gradient, each
        in autograd's operation order, and a sum of two terms does not depend on the order autograd adds them in.  This is
        the perceptual path (d_perc scaled by disc_wt, the g plan's input gradient added in gen_loss_grad_kernel);
      * with the sync term, the expert's embedding gradient is computed by cosine_bce_bwd_kernel, not by torch's
        cosine_similarity backward, so dL/dg differs in its last bits, and the backward through the generator's
        batch-statistics BatchNorms amplifies that (tests/test_precision_model.py): the head and the output block stay
        within fp32 rounding (measured <= 5.2e-6 relative L2), the deeper tensors within a few per cent (median 1.1e-2,
        max 1.7e-2)."""
    from wav2lip_b200.training import HQWav2LipTrainStep
    B, T, WD = 8, 5, 0.07
    x, indiv_mels, mel, gt = (t.cuda() for t in _train_inputs(B, seed=12))
    ma, da, sa = _nets()
    for p in sa.parameters():
        p.requires_grad = False
    g = ma(indiv_mels, x)                                                   # the bridge, in the script's order (:225-253)
    if ws > 0:
        half = g[:, :, :, g.size(3) // 2:]
        a, v = sa(mel, torch.cat([half[:, :, i] for i in range(T)], dim=1))
        sync = F.binary_cross_entropy(F.cosine_similarity(a, v).unsqueeze(1), torch.ones(B, 1, device=g.device))
    else:
        sync = 0.
    pf = da(g)
    perceptual = F.binary_cross_entropy(pf, torch.ones_like(pf))
    l1 = F.l1_loss(g, gt)
    loss = ws * sync + WD * perceptual + (1. - ws - WD) * l1
    loss.backward()
    gen_ref = {n: p.grad.clone() for n, p in ma.named_parameters()}
    for p in da.parameters():
        p.grad = None                                                       # disc_optimizer.zero_grad() (:245)
    pr = da(gt)
    real = F.binary_cross_entropy(pr, torch.ones_like(pr))
    real.backward()
    pf_det = da(g.detach())
    fake = F.binary_cross_entropy(pf_det, torch.zeros_like(pf_det))
    fake.backward()
    disc_ref = {n: p.grad.clone() for n, p in da.named_parameters()}
    sync_v = float(sync) if ws == 0 else sync.item()
    ref = np.array([sync_v, l1.item(), perceptual.item(), loss.item(), real.item(), fake.item()])
    mb, db, sb = _nets()
    step = HQWav2LipTrainStep(mb, db, sb, syncnet_wt=ws, disc_wt=WD)
    lo = step(x, indiv_mels, mel, gt).cpu().numpy()
    gf = step.last_output()
    same_g = bool(torch.equal(gf, g.detach()))
    _, dc, _ = _nets()
    pf2 = dc(gf)                           # the step's own g through an untouched discriminator's training forward
    fake2 = F.binary_cross_entropy(pf2, torch.zeros_like(pf2)).item()
    rel = np.abs(lo - ref) / np.maximum(np.abs(ref), 1e-30)
    gen_err = {n: rel_l2(step.b.grads[n], r) for n, r in gen_ref.items() if r.norm().item() > 0}
    gen_same = [n for n, r in gen_ref.items() if torch.equal(step.b.grads[n], r)]
    disc_diff = [n for n, r in disc_ref.items() if not torch.equal(step.db.grads[n], r)]
    head = ["output_block.1.weight", "output_block.1.bias", "output_block.0.conv_block.0.weight"]
    report(f"hq_fused_vs_bridge_ws{ws}", {"same_g": same_g, "losses": lo.tolist(), "bridge": ref.tolist(), "rel": rel.tolist(),
                                          "fake_on_own_g": fake2, "gen_bit_identical": f"{len(gen_same)}/{len(gen_ref)}",
                                          "disc_not_identical": disc_diff, "gen_grad": summarize(gen_err),
                                          "gen_grad_head": {n: gen_err.get(n) for n in head}})
    assert same_g
    assert rel.max() <= 1e-6, rel
    assert abs(lo[5] - fake2) <= 1e-6 * fake2
    assert not disc_diff, disc_diff
    if ws == 0:
        assert len(gen_same) == len(gen_ref), sorted(set(gen_ref) - set(gen_same))[:8]
    else:
        assert all(gen_err[n] <= 1e-4 for n in head), {n: gen_err[n] for n in head}
        assert max(gen_err.values()) <= 0.05, summarize(gen_err)


# ----------------------------------------------------------------------------------------------------------------------
# color_syncnet_train.py
# ----------------------------------------------------------------------------------------------------------------------
def test_syncnet_fused_step_against_the_reference_golden(golden_dir):
    """Two iterations of color_syncnet_train.py:149-163 (B = 4, y = [1,0,1,0]) against the REAL script (train.npz sync0/1)."""
    from wav2lip_b200.training import SyncNetTrainStep
    gold = np.load(os.path.join(golden_dir, "train.npz"))
    model = _syncnet(O.make_state_dict("syncnet", 2, init="default"))
    mel, face = O.make_syncnet_inputs(4, seed=5)
    y = torch.tensor([[1.0], [0.0], [1.0], [0.0]])
    step = SyncNetTrainStep(model, lr=1e-4)
    for it in range(2):
        loss = step(face.cuda(), mel.cuda(), y.cuda()).item()
        ref = float(gold[f"sync{it}_loss"][0])
        names = list(gold[f"sync{it}_sd_names"])
        assert names == list(model.state_dict().keys())
        rel = _sd_rel(model, gold[f"sync{it}_sd_fp"])
        is_stat = np.array([("running" in n) or ("num_batches" in n) for n in names])
        report(f"syncnet_fused_step{it}", {"loss": loss, "ref": ref, "loss_rel": abs(loss - ref) / ref,
                                           "sd_rel_max": float(rel[~is_stat].max()), "stat_rel_max": float(rel[is_stat].max())})
        # the loss: cosine of two embeddings through BatchNorms over B = 4 samples — bf16 moves it by per cents
        assert abs(loss - ref) <= 0.12 * ref, (it, loss, ref)
        assert rel[~is_stat].max() <= 6e-3, (it, rel[~is_stat].max())
        assert rel[is_stat].max() <= 6e-2, (it, rel[is_stat].max())


def test_syncnet_fused_step_gradients_against_float64_autograd():
    """Every parameter gradient of the fused expert step against float64 autograd (all ReLUs active, B = 16), with the
    bars of the bridge's test_syncnet_training_through_autograd_bridge."""
    from wav2lip_b200.training import SyncNetTrainStep
    sd = relu_active(O.make_state_dict("syncnet", 2, init="default"))
    mel, face = O.make_syncnet_inputs(16, seed=5)
    y = torch.tensor([[1.0], [0.0]] * 8)
    leaves = {k: v.double().clone().requires_grad_(k.endswith(".weight") or k.endswith(".bias"))
              for k, v in sd.items() if v.dtype.is_floating_point}
    a, v = O.syncnet_forward(leaves, mel.double(), face.double(), training=True)
    lref = F.binary_cross_entropy(F.cosine_similarity(a, v).unsqueeze(1), y.double())
    names = [k for k, t in leaves.items() if t.requires_grad]
    ref = dict(zip(names, torch.autograd.grad(lref, [leaves[k] for k in names])))
    model = _syncnet(sd)
    step = SyncNetTrainStep(model, lr=1e-4)
    loss = step(face.cuda(), mel.cuda(), y.cuda()).item()
    scale = max(g.norm().item() for g in ref.values())
    errs = {n: rel_l2(step.b.grads[n], ref[n]) for n in names
            if not n.endswith("conv_block.0.bias") and ref[n].norm().item() >= 1e-6 * scale}
    rep = summarize(errs)
    rep.update({"loss": loss, "ref_loss": lref.item()})
    report("syncnet_fused_f64", rep)
    assert all(float(step.b.grads[n].abs().max()) == 0.0 for n in names if n.endswith("conv_block.0.bias"))
    assert rep["max"] <= 1.0 and rep["p90"] <= 0.35 and rep["median"] <= 0.25 and rep["n"] >= 60, rep


# ----------------------------------------------------------------------------------------------------------------------
# optimizer state
# ----------------------------------------------------------------------------------------------------------------------
def _make_steps(kind):
    """(step, [(module, binding, betas, export, load)]) for one of the three fused steps, at a small batch."""
    from wav2lip_b200.training import HQWav2LipTrainStep, SyncNetTrainStep, Wav2LipTrainStep
    if kind == "sync":
        model = _syncnet(O.make_state_dict("syncnet", 2, init="default"))
        step = SyncNetTrainStep(model, lr=1e-4)
        mel, face = O.make_syncnet_inputs(4, seed=5)
        args = (face.cuda(), mel.cuda(), torch.tensor([[1.0], [0.0], [1.0], [0.0]]).cuda())
        return step, args, [(model, step.b, (0.9, 0.999), step.optimizer_state_dict, step.load_optimizer_state_dict)]
    model, disc, syncnet = _nets()
    args = tuple(t.cuda() for t in _train_inputs(2, seed=8))
    if kind == "wav2lip":
        step = Wav2LipTrainStep(model, syncnet, lr=1e-4, syncnet_wt=0.03)
        return step, args, [(model, step.b, (0.9, 0.999), step.optimizer_state_dict, step.load_optimizer_state_dict)]
    step = HQWav2LipTrainStep(model, disc, syncnet, syncnet_wt=0.03, disc_wt=0.07)
    return step, args, [(model, step.b, (0.5, 0.999), step.optimizer_state_dict, step.load_optimizer_state_dict),
                        (disc, step.db, (0.5, 0.999), step.disc_optimizer_state_dict, step.load_disc_optimizer_state_dict)]


def _params(module):
    return {n: p.detach().clone() for n, p in module.named_parameters()}


def _torch_next(before, sd, grads, lr):
    """torch.optim.Adam loaded with sd, stepped once on `grads` from the parameters `before`."""
    names = list(before)
    ps = [before[n].clone().requires_grad_(True) for n in names]
    opt = torch.optim.Adam(ps, lr=lr, betas=tuple(sd["param_groups"][0]["betas"]))
    opt.load_state_dict(copy.deepcopy(sd))
    for p, n in zip(ps, names):
        p.grad = grads[n].clone()
    opt.step()
    return {n: p.detach() for n, p in zip(names, ps)}


def _update_err(module, before, want, lr):
    """max over elements of |fused - torch| in units of the bar 1e-3 lr + one fp32 ulp of the parameter (the two
    implementations round p - update separately)."""
    worst = 0.0
    for n in before:
        got = module.get_parameter(n).detach()
        bar = 1e-3 * lr + torch.finfo(torch.float32).eps * before[n].abs()
        worst = max(worst, ((got - want[n]).abs() / bar).max().item())
    return worst


@pytest.mark.parametrize("kind", ["wav2lip", "hq", "sync"])
def test_optimizer_state_is_torch_adams(kind):
    """After one fused step the exported moments are (1-b1) g and (1-b2) g g in fp32, step 1; torch's Adam loaded with that
    export and stepped on the next gradients lands on the fused step's next parameters; a state torch's Adam wrote after
    k = 3 steps loads into a fresh fused step, exports back bit for bit, and the next update uses step k + 1."""
    step, args, nets = _make_steps(kind)
    step(*args)
    exported = []
    for module, b, betas, export, _ in nets:
        sd = export()
        exported.append(sd)
        names = [n for n, _ in module.named_parameters()]
        assert sorted(sd["state"]) == list(range(len(names)))
        c1 = torch.tensor(1.0) - torch.tensor(betas[0])
        c2 = torch.tensor(1.0) - torch.tensor(betas[1])
        for i, n in enumerate(names):
            g = b.grads[n]
            st = sd["state"][i]
            assert float(st["step"]) == 1.0
            assert torch.equal(st["exp_avg"], c1.cuda() * g), n
            assert torch.equal(st["exp_avg_sq"], (c2.cuda() * g) * g), n
        assert sd["param_groups"][0]["betas"] == betas and sd["param_groups"][0]["params"] == list(range(len(names)))
    before = [_params(m) for m, *_ in nets]
    step(*args)
    for (module, b, betas, _, _), sd, p0 in zip(nets, exported, before):
        want = _torch_next(p0, sd, {n: b.grads[n] for n in p0}, 1e-4)
        err = _update_err(module, p0, want, 1e-4)
        report(f"adam_next_{kind}_{module.NET}", {"err_over_bar": err})
        assert err <= 1.0, err
    # a state torch's Adam wrote after 3 steps, into a fresh fused step
    step2, args2, nets2 = _make_steps(kind)
    gen = torch.Generator(device="cuda").manual_seed(3)
    loaded = []
    for module, b, betas, export, load in nets2:
        ps = [p.detach().clone().requires_grad_(True) for p in module.parameters()]
        opt = torch.optim.Adam(ps, lr=1e-4, betas=betas)
        for _ in range(3):
            for p in ps:
                p.grad = torch.randn(p.shape, device=p.device, generator=gen) * 1e-3
            opt.step()
        sd = opt.state_dict()
        load(copy.deepcopy(sd))
        back = export()
        assert sorted(back["state"]) == sorted(sd["state"])
        for i in sd["state"]:
            assert float(back["state"][i]["step"]) == 3.0
            assert torch.equal(back["state"][i]["exp_avg"], sd["state"][i]["exp_avg"])
            assert torch.equal(back["state"][i]["exp_avg_sq"], sd["state"][i]["exp_avg_sq"])
        loaded.append(sd)
    before = [_params(m) for m, *_ in nets2]
    step2(*args2)
    for (module, b, betas, export, _), p0, sd in zip(nets2, before, loaded):
        want = _torch_next(p0, sd, {n: b.grads[n] for n in p0}, 1e-4)
        err = _update_err(module, p0, want, 1e-4)
        report(f"adam_loaded_next_{kind}_{module.NET}", {"err_over_bar": err})
        assert err <= 1.0, err
        assert float(export()["state"][0]["step"]) == 4.0


# ----------------------------------------------------------------------------------------------------------------------
# determinism, guards
# ----------------------------------------------------------------------------------------------------------------------
def _run_twice_state(kind):
    """Two iterations of a fresh step from fixed weights: every output that must not depend on timing."""
    step, args, nets = _make_steps(kind)
    losses = [step(*args).clone() for _ in range(2)]
    out = {"losses": torch.stack(losses).cpu()}
    for module, b, betas, export, _ in nets:
        for k, v in module.state_dict().items():
            out[f"{module.NET}:{k}"] = v.detach().cpu().clone()
        sd = export()
        for i, st in sd["state"].items():
            out[f"{module.NET}:m{i}"] = st["exp_avg"].cpu()
            out[f"{module.NET}:v{i}"] = st["exp_avg_sq"].cpu()
    if kind == "hq":
        for k, v in step.syncnet.state_dict().items():
            out[f"expert:{k}"] = v.detach().cpu().clone()
    return out


@pytest.mark.parametrize("kind", ["hq", "sync"])
def test_fused_steps_are_deterministic_across_runs_and_stream_switches(kind, monkeypatch):
    ref = _run_twice_state(kind)
    runs = {"again": {}, "W2L_DISABLE_WGSTREAM": {"W2L_DISABLE_WGSTREAM": "1"}, "W2L_DISABLE_AUXSTREAM": {"W2L_DISABLE_AUXSTREAM": "1"}}
    for label, env in runs.items():
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            got = _run_twice_state(kind)       # new modules: new contexts, which read the switches
        assert got.keys() == ref.keys()
        diff = [k for k in ref if not torch.equal(got[k], ref[k])]
        assert not diff, (label, diff[:8])


def test_fused_steps_refuse_bad_inputs_before_launching_anything():
    from wav2lip_b200 import _lib
    from wav2lip_b200.training import HQWav2LipTrainStep, SyncNetTrainStep, Wav2LipTrainStep
    model, disc, syncnet = _nets()
    step = HQWav2LipTrainStep(model, disc, syncnet, syncnet_wt=0.03, disc_wt=0.07)
    x, indiv_mels, mel, gt = (t.cuda() for t in _train_inputs(2, seed=8))
    p0 = _params(model)
    n0 = step.b.ctx.launch_count()
    with pytest.raises(_lib.W2LError):
        step(x.cpu(), indiv_mels, mel, gt)                                  # a CPU tensor
    with pytest.raises(ValueError):
        step(x[:, :3], indiv_mels, mel, gt)                                  # wrong shape
    with pytest.raises(ValueError):
        step(x, indiv_mels, mel[:, :, :40], gt)
    with pytest.raises(_lib.W2LError):
        step(x, indiv_mels, None, gt)                                        # syncnet_wt > 0 without mel
    x3, im3, _, gt3 = (t.cuda() for t in _train_inputs(2, seed=8, T=3))
    with pytest.raises(_lib.W2LError):
        step(x3, im3, mel, gt3)                                              # syncnet_wt > 0 needs T = 5
    m2, _, _ = _nets()
    plain = Wav2LipTrainStep(m2, None)                                       # a context without a bound discriminator
    b = plain.b
    n_plain = b.ctx.launch_count()
    with pytest.raises(_lib.W2LError):
        _lib.check(b.ctx.lib.w2l_hq_wav2lip_train_step(b.ctx.h, _P(indiv_mels), _P(x), None, _P(gt), 2, 5, 0.0, 0.07, 1e-4, 1e-4,
                                                       None, None))
    s = SyncNetTrainStep(_syncnet(O.make_state_dict("syncnet", 2, init="default")))
    smel, sface = (t.cuda() for t in O.make_syncnet_inputs(4, seed=5))
    n_sync = s.b.ctx.launch_count()
    with pytest.raises(ValueError):
        s(sface, smel, torch.ones(4).cuda())                                 # y must be (B, 1)
    with pytest.raises(_lib.W2LError):
        s(sface.cpu(), smel, torch.ones(4, 1).cuda())
    torch.cuda.synchronize()
    assert step.b.ctx.launch_count() == n0 and b.ctx.launch_count() == n_plain and s.b.ctx.launch_count() == n_sync
    assert all(torch.equal(p0[n], p.detach()) for n, p in model.named_parameters())


def _P(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr())


# ----------------------------------------------------------------------------------------------------------------------
# two GPUs
# ----------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _dp_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from wav2lip_b200.training import HQWav2LipTrainStep, SyncNetTrainStep, init_data_parallel

        def avg(t):
            t = t.clone()
            dist.all_reduce(t)
            return t / world

        def err(a, b):
            return float((a - b).norm() / b.norm())
        x, im, mel, gt = (t.cuda(rank) for t in _train_inputs(2, seed=50 + rank))    # different data on every rank
        res = {}
        for dp in (False, True):
            model, disc, syncnet = _nets()
            st = HQWav2LipTrainStep(model.cuda(rank), disc.cuda(rank), syncnet.cuda(rank), syncnet_wt=0.03, disc_wt=0.07)
            if dp:
                assert init_data_parallel(st) == world
            st(x, im, mel, gt)
            torch.cuda.synchronize()
            res[dp] = (st.b.arena.clone(), st.db.arena.clone())
        res_g = err(res[True][0], avg(res[False][0]))
        res_d = err(res[True][1], avg(res[False][1]))
        mel_s, face_s = O.make_syncnet_inputs(4, seed=60 + rank)
        y = torch.tensor([[1.0], [0.0], [1.0], [0.0]]).cuda(rank)
        sres = {}
        for dp in (False, True):
            s = SyncNetTrainStep(_syncnet(O.make_state_dict("syncnet", 2, init="default")).cuda(rank))
            if dp:
                init_data_parallel(s)
            s(face_s.cuda(rank), mel_s.cuda(rank), y)
            torch.cuda.synchronize()
            sres[dp] = s.b.arena.clone()
        res_s = err(sres[True], avg(sres[False]))
        local = err(res[False][1], res[True][1])
        q.put((rank, res_g, res_d, res_s, local))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_fused_steps_all_reduce_every_networks_gradients():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=900) for _ in range(2)]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, eg, ed, es, local in res:
        assert eg <= 1e-5 and ed <= 1e-5 and es <= 1e-5, (rank, eg, ed, es)
        assert local > 1e-2, rank                       # the ranks had different gradients before the collective
