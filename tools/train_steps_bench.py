"""Time the fused training steps against the autograd bridge, on one GPU in one process:

  hq      hq_wav2lip_train.py:212-256 — HQWav2LipTrainStep vs the script's statements on the mirrors (two torch Adams),
          B = 16 (hparams.batch_size) and B = 64, T = 5, syncnet_wt 0.03, disc_wt 0.07;
  wav2lip Wav2LipTrainStep at the same B (the discriminator's marginal cost is hq - wav2lip);
  expert  color_syncnet_train.py:149-163 — SyncNetTrainStep vs the script's statements, B = 64 (syncnet_batch_size).

The two versions of a row alternate (--rounds rounds of --warmup + --iters iterations each); a round's time is the median
of its iterations, each ended by a device synchronise; the table gives the median over rounds and the range.  Before timing,
step 0 of both versions runs on identical fresh weights; the run stops with an error if their losses differ by more than
1e-5 relative.  The card's name, power limit and SM
clock are read in the same run.  TFLOP/s are algorithmic: convolution FLOPs of the forward (w2l_train_flops) times the
passes each step needs (3 for a network with weight and input gradients, 2 for a forward + input gradient only), for the
fused step's own passes — the bridge does the same useful work plus what the fused step saves.

    python tools/train_steps_bench.py [--rounds 3] [--warmup 5] [--iters 20] [--json out.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import w2l_oracle as O  # noqa: E402
from wav2lip_b200 import _lib  # noqa: E402
from wav2lip_b200.models import SyncNet_color, Wav2Lip, Wav2Lip_disc_qual  # noqa: E402
from wav2lip_b200.training import HQWav2LipTrainStep, SyncNetTrainStep, Wav2LipTrainStep  # noqa: E402

T, WS, WD = 5, 0.03, 0.07


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def nets(dev):
    m, d, s = Wav2Lip(), Wav2Lip_disc_qual(), SyncNet_color()
    m.load_state_dict(O.make_state_dict("generator", 0, init="default"))
    d.load_state_dict(O.make_state_dict("disc", 3, init="default"))
    s.load_state_dict(O.make_state_dict("syncnet", 1, init="default"))
    return m.to(dev).train(), d.to(dev).train(), s.to(dev).train()


def gen_batch(B, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, 6, T, 96, 96), generator=g)
    im = torch.rand((B, T, 1, 80, 16), generator=g) * 8 - 4
    mel = torch.rand((B, 1, 80, 16), generator=g) * 8 - 4
    gt = torch.rand((B, 3, T, 96, 96), generator=g)
    return x.to(dev), im.to(dev), mel.to(dev), gt.to(dev)


def sync_batch(B, dev, seed=0):
    mel, face = O.make_syncnet_inputs(B, seed=seed)
    y = torch.tensor([[float(i % 2)] for i in range(B)])
    return face.to(dev), mel.to(dev), y.to(dev)


def hq_bridge(model, disc, syncnet):
    """hq_wav2lip_train.py:212-256 as the script writes it, on the mirrors."""
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-4, betas=(0.5, 0.999))
    dopt = torch.optim.Adam([p for p in disc.parameters() if p.requires_grad], lr=1e-4, betas=(0.5, 0.999))
    for p in syncnet.parameters():
        p.requires_grad = False

    def it(x, im, mel, gt):
        disc.train(); model.train()
        opt.zero_grad(); dopt.zero_grad()
        g = model(im, x)
        half = g[:, :, :, g.size(3) // 2:]
        a, v = syncnet(mel, torch.cat([half[:, :, i] for i in range(T)], dim=1))
        sync = F.binary_cross_entropy(F.cosine_similarity(a, v).unsqueeze(1), torch.ones(g.size(0), 1, device=g.device))
        perceptual = disc.perceptual_forward(g)
        l1 = F.l1_loss(g, gt)
        loss = WS * sync + WD * perceptual + (1 - WS - WD) * l1
        loss.backward()
        opt.step()
        dopt.zero_grad()
        pr = disc(gt)
        real = F.binary_cross_entropy(pr, torch.ones_like(pr))
        real.backward()
        pf = disc(g.detach())
        fake = F.binary_cross_entropy(pf, torch.zeros_like(pf))
        fake.backward()
        dopt.step()
        return torch.stack([sync, l1, perceptual, loss, real, fake]).detach()
    return it


def sync_bridge(model):
    """color_syncnet_train.py:149-163 as the script writes it, on the mirror."""
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-4)

    def it(x, mel, y):
        model.train()
        opt.zero_grad()
        a, v = model(mel, x)
        loss = F.binary_cross_entropy(F.cosine_similarity(a, v).unsqueeze(1), y)
        loss.backward()
        opt.step()
        return loss.detach().reshape(1)
    return it


def time_iters(fn, args, n):
    ts = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(*args)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def alternate(versions, args, rounds, warmup, iters):
    res = {k: [] for k in versions}
    for _ in range(rounds):
        for k, fn in versions.items():
            for _ in range(warmup):
                fn(*args)
            res[k].append(time_iters(fn, args, iters))
    return {k: (statistics.median(v), min(v), max(v)) for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_steps_bench.py measures on a CUDA device; none found")
    dev = torch.device("cuda", 0)
    out = {"card (name, power limit, SM clock, max SM clock) before": card(), "rows": []}
    print(out["card (name, power limit, SM clock, max SM clock) before"], flush=True)

    # ---- step 0 of both versions on identical fresh weights ----
    args = gen_batch(16, dev, seed=1)
    ref = hq_bridge(*nets(dev))(*args)
    m, d, s = nets(dev)
    got = HQWav2LipTrainStep(m, d, s, syncnet_wt=WS, disc_wt=WD)(*[args[i] for i in (0, 1, 2, 3)])
    rel = ((got - ref).abs() / ref.abs()).max().item()
    sargs = sync_batch(64, dev, seed=2)
    sd = O.make_state_dict("syncnet", 2, init="default")
    s1, s2 = SyncNet_color(), SyncNet_color()
    s1.load_state_dict(sd); s2.load_state_dict(sd)
    sref = sync_bridge(s1.to(dev).train())(*sargs)
    sgot = SyncNetTrainStep(s2.to(dev).train())(*sargs)
    srel = ((sgot - sref).abs() / sref.abs()).max().item()
    out["step0"] = {"hq_losses_fused": got.tolist(), "hq_losses_bridge": ref.tolist(), "hq_max_rel": rel,
                    "expert_loss_fused": sgot.item(), "expert_loss_bridge": sref.item(), "expert_rel": srel}
    print("step 0:", json.dumps(out["step0"]), flush=True)
    # same plans and kernels: only the loss arithmetic's rounding may differ (measured 1.1e-7 on an H100)
    if not (rel <= 1e-5 and srel <= 1e-5):
        raise SystemExit(f"step 0: the fused and bridge losses disagree (hq {rel:.3g}, expert {srel:.3g} relative; bar 1e-5)")

    # ---- timing ----
    for B in (16, 64):
        model, disc, syncnet = nets(dev)
        fused = HQWav2LipTrainStep(model, disc, syncnet, syncnet_wt=WS, disc_wt=WD)
        plain = Wav2LipTrainStep(model, syncnet, syncnet_wt=WS)
        bridge = hq_bridge(*nets(dev))
        args = gen_batch(B, dev, seed=3)
        r = alternate({"hq fused": fused, "hq bridge": bridge, "wav2lip fused": plain}, args, a.rounds, a.warmup, a.iters)
        ctx = fused.b.ctx
        fg, fs, fd = (ctx.lib.w2l_train_flops(ctx.h, n) for n in (_lib.NET_GENERATOR, _lib.NET_SYNCNET, _lib.NET_DISC))
        flops_hq = 3 * fg + 2 * fs + 7 * fd      # disc: 2 forwards, perceptual dgrad, real and fake dgrad + wgrad
        flops_w2l = 3 * fg + 2 * fs
        for k, (med, lo, hi) in r.items():
            fl = flops_w2l if k.startswith("wav2lip") else flops_hq
            row = {"row": k, "B": B, "T": T, "ms": round(med, 2), "ms_range": [round(lo, 2), round(hi, 2)],
                   "crops_per_s": round(B * T / med * 1e3), "tflops_algorithmic": round(fl / med * 1e-9, 1)}
            out["rows"].append(row)
            print(json.dumps(row), flush=True)
        out[f"device_bytes_generator_context_B{B}"] = ctx.device_bytes()
        del fused, plain, bridge, model, disc, syncnet
        torch.cuda.empty_cache()
    s1, s2 = SyncNet_color(), SyncNet_color()
    s1.load_state_dict(sd); s2.load_state_dict(sd)
    fused = SyncNetTrainStep(s1.to(dev).train())
    bridge = sync_bridge(s2.to(dev).train())
    r = alternate({"expert fused": fused, "expert bridge": bridge}, sargs, a.rounds, a.warmup, a.iters)
    ctx = fused.b.ctx
    fl = 3 * ctx.lib.w2l_train_flops(ctx.h, _lib.NET_SYNCNET)
    for k, (med, lo, hi) in r.items():
        row = {"row": k, "B": 64, "ms": round(med, 2), "ms_range": [round(lo, 2), round(hi, 2)],
               "windows_per_s": round(64 / med * 1e3), "tflops_algorithmic": round(fl / med * 1e-9, 1)}
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    out["device_bytes_expert_context"] = ctx.device_bytes()
    out["card (name, power limit, SM clock, max SM clock) after"] = card()
    print(out["card (name, power limit, SM clock, max SM clock) after"], flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
