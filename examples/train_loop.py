"""The training loops of the reference on the H100 core, on synthetic batches or a preprocessed dataset:

  --mode script   the statements of wav2lip_train.py:210-231 as the script writes them — `model.train()`, `g = model(indiv_mels, x)`,
                  `get_sync_loss` through the frozen expert (left in train mode, :187-189), `recon_loss`, `loss.backward()`,
                  `torch.optim.Adam.step()` — on the mirrors: the forward/backward of each network is one native call behind
                  an autograd node (wav2lip_b200/training.py), torch only does the loss arithmetic;
  --mode fused    the same iteration as ONE native call (`Wav2LipTrainStep` -> w2l_wav2lip_train_step): forward, losses,
                  backward, bucketed gradient all-reduce (when launched under torchrun), Adam;
  --mode hq       hq_wav2lip_train.py:213-255: generator + perceptual loss through the quality discriminator + the
                  discriminator's real/fake step, two Adam optimizers (betas 0.5, 0.999), through the autograd bridge;
  --mode hq-fused the same iteration as ONE native call (`HQWav2LipTrainStep` -> w2l_hq_wav2lip_train_step), both
                  networks' gradients all-reduced under torchrun;
  --mode expert   color_syncnet_train.py:149-163, the expert's own training, as ONE native call (`SyncNetTrainStep` ->
                  w2l_syncnet_train_step); with --data-root the batches are SyncNetBatches'.

--save F writes the fused modes' optimizer state after the last iteration as the reference's checkpoints store it
(`optimizer.state_dict()`, torch.optim.Adam's format) and --resume F loads it before the first one.

With --data-root DIR (a preprocess.py-layout dataset) the batches are the reference Dataset's, assembled on the device from a
cache built once (wav2lip_b200/data.py: TrainDataCache + Wav2LipBatches); the video list is filelists/train.txt relative to the
current directory, as hparams.get_image_list reads it, or --filelist F.  Without it the batches are synthetic.

Run:  python examples/train_loop.py --mode fused --iters 20 --batch 16
      python examples/train_loop.py --mode fused --data-root DIR [--filelist F]
      python examples/train_loop.py --mode expert --data-root DIR --batch 64
      python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 examples/train_loop.py --mode fused
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F
from torch import nn, optim

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2lip_b200.models import SyncNet_color, Wav2Lip, Wav2Lip_disc_qual  # noqa: E402
from wav2lip_b200.training import HQWav2LipTrainStep, SyncNetTrainStep, Wav2LipTrainStep, init_data_parallel  # noqa: E402

syncnet_T = 5            # hparams.py
SYNCNET_WT, DISC_WT = 0.03, 0.07


def batch(B, dev, seed):
    """x (B,6,T,96,96), indiv_mels (B,T,1,80,16), mel (B,1,80,16), gt (B,3,T,96,96) as the Dataset builds them
    (wav2lip_train.py:153-163)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B, 6, syncnet_T, 96, 96), generator=g)
    indiv_mels = torch.rand((B, syncnet_T, 1, 80, 16), generator=g) * 8 - 4
    mel = torch.rand((B, 1, 80, 16), generator=g) * 8 - 4
    gt = torch.rand((B, 3, syncnet_T, 96, 96), generator=g)
    return x.to(dev), indiv_mels.to(dev), mel.to(dev), gt.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["script", "fused", "hq", "hq-fused", "expert"], default="fused")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--data-root", default=None, help="train on this preprocessed dataset instead of synthetic batches")
    ap.add_argument("--filelist", default=None, help="video list (default: filelists/train.txt in the current directory)")
    ap.add_argument("--save", default=None, help="fused modes: write the optimizer state here after the last iteration")
    ap.add_argument("--resume", default=None, help="fused modes: load the optimizer state from here first")
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)

    torch.manual_seed(0)                                   # the same initial weights on every rank
    model = Wav2Lip().to(dev)
    syncnet = SyncNet_color().to(dev)
    for p in syncnet.parameters():
        p.requires_grad = False                            # wav2lip_train.py:188-189
    logloss, recon_loss = nn.BCELoss(), nn.L1Loss()

    def get_sync_loss(mel, g):                             # wav2lip_train.py:192-198
        g = g[:, :, :, g.size(3) // 2:]
        g = torch.cat([g[:, :, i] for i in range(syncnet_T)], dim=1)
        a, v = syncnet(mel, g)
        d = F.cosine_similarity(a, v)
        return logloss(d.unsqueeze(1), torch.ones(g.size(0), 1, device=g.device))

    step = None
    if args.mode == "fused":
        step = Wav2LipTrainStep(model.train(), syncnet.train(), lr=1e-4, syncnet_wt=SYNCNET_WT)
    elif args.mode == "hq-fused":
        step = HQWav2LipTrainStep(model.train(), Wav2Lip_disc_qual().to(dev).train(), syncnet.train(), lr=1e-4, disc_lr=1e-4,
                                  syncnet_wt=SYNCNET_WT, disc_wt=DISC_WT)
    elif args.mode == "expert":
        expert = SyncNet_color().to(dev).train()
        step = SyncNetTrainStep(expert, lr=1e-4)
    elif args.mode == "script":
        optimizer = optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-4)          # :357-360
    else:
        disc = Wav2Lip_disc_qual().to(dev)
        optimizer = optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-4, betas=(0.5, 0.999))
        disc_optimizer = optim.Adam([p for p in disc.parameters() if p.requires_grad], lr=1e-4, betas=(0.5, 0.999))

    if step is not None:
        if world > 1:
            init_data_parallel(step)
        if args.resume:
            ck = torch.load(args.resume, map_location=dev)
            step.load_optimizer_state_dict(ck["optimizer"])
            if "disc_optimizer" in ck:
                step.load_disc_optimizer_state_dict(ck["disc_optimizer"])

    feed = None
    if args.data_root is not None:
        from wav2lip_b200.data import SyncNetBatches, TrainDataCache, Wav2LipBatches
        cache = TrainDataCache.from_data_root(args.data_root, "train", filelist=args.filelist, device=dev)
        feed = (SyncNetBatches if args.mode == "expert" else Wav2LipBatches)(cache, args.batch)
        if rank == 0:
            print(f"dataset: {len(cache.videos)} videos, {cache.n_frames} frames, {cache.n_mel_rows} mel rows", flush=True)

    t0 = None
    for it in range(args.iters):
        if it == 2:
            torch.cuda.synchronize(); t0 = time.time()
        if args.mode == "expert":
            if feed is not None:
                x, mel, y = feed.next_batch()
            else:
                x = torch.rand((args.batch, 3 * syncnet_T, 48, 96), device=dev)
                mel = torch.rand((args.batch, 1, 80, 16), device=dev) * 8 - 4
                y = (torch.rand((args.batch, 1), device=dev) > 0.5).float()
            loss = step(x, mel, y).item()
            if rank == 0:
                print(f"iter {it}: loss {loss:.4f}", flush=True)
            continue
        if feed is not None:
            x, indiv_mels, mel, gt = feed.next_batch()
        else:
            x, indiv_mels, mel, gt = batch(args.batch, dev, seed=1000 * rank + it)
        if args.mode == "fused":
            sync_loss, l1, _, loss = step(x, indiv_mels, mel, gt).tolist()
        elif args.mode == "hq-fused":
            sync_loss, l1, _, loss, _, _ = step(x, indiv_mels, mel, gt).tolist()
        elif args.mode == "script":
            model.train(); optimizer.zero_grad()                                                     # :210-212
            g = model(indiv_mels, x)
            sync_loss = get_sync_loss(mel, g)
            l1 = recon_loss(g, gt)
            loss = SYNCNET_WT * sync_loss + (1 - SYNCNET_WT) * l1
            loss.backward(); optimizer.step()
            sync_loss, l1, loss = sync_loss.item(), l1.item(), loss.item()
        else:
            disc.train(); model.train()                                                              # hq :213-214
            optimizer.zero_grad(); disc_optimizer.zero_grad()
            g = model(indiv_mels, x)
            sync_loss = get_sync_loss(mel, g)
            perceptual = disc.perceptual_forward(g)                                                   # :233
            l1 = recon_loss(g, gt)
            loss = SYNCNET_WT * sync_loss + DISC_WT * perceptual + (1. - SYNCNET_WT - DISC_WT) * l1
            loss.backward(); optimizer.step()
            disc_optimizer.zero_grad()                                                                # :245
            pred = disc(gt)
            F.binary_cross_entropy(pred, torch.ones((len(pred), 1), device=dev)).backward()
            pred = disc(g.detach())
            F.binary_cross_entropy(pred, torch.zeros((len(pred), 1), device=dev)).backward()
            disc_optimizer.step()
            sync_loss, l1, loss = sync_loss.item(), l1.item(), loss.item()
        if rank == 0:
            print(f"iter {it}: loss {loss:.4f}  l1 {l1:.4f}  sync {sync_loss:.4f}", flush=True)
    torch.cuda.synchronize()
    if rank == 0 and t0 is not None and args.iters > 2:
        dt = (time.time() - t0) / (args.iters - 2)
        per = 1 if args.mode == "expert" else syncnet_T
        print(f"{dt * 1e3:.1f} ms per iteration, {world * args.batch * per / dt:.0f} samples/s trained ({world} GPU(s), B={args.batch}/GPU)")
    if step is not None and args.save and rank == 0:
        ck = {"optimizer": step.optimizer_state_dict()}
        if args.mode == "hq-fused":
            ck["disc_optimizer"] = step.disc_optimizer_state_dict()
        torch.save(ck, args.save)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
