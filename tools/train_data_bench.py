"""Training data pipeline timing (wav2lip_b200/data.py): the batch gather kernels, the host sampler, the training step fed by
`Wav2LipBatches`, and a restatement of the reference's per-sample loader on the same host.

    python tools/train_data_bench.py [--videos 64] [--frames 120] [--iters 200] [--train-iters 30] [--out FILE]
    python tools/train_data_bench.py --make-dataset DIR [--videos 8] [--frames 60]    # only write a dataset

It writes a preprocessed dataset (96..160-pixel jpg crops named <id>.jpg and a 16 kHz audio.wav per video, plus
DIR/filelists/train.txt) to a temporary directory and builds the cache from it with `TrainDataCache.from_data_root`.
One JSON object is printed (and written to --out):
  card                       nvidia-smi name, power limit and max SM clock, read in the same run
  cache_build_s              from_data_root wall time (decode on 16 threads, device resize, device mel)
  gather[storage][net][B]    kernel time per launch from torch.profiler (a run of its own), the bytes the gather must move
                             (frames read, mel rows read, outputs written) and bytes / kernel time against 3.35 TB/s (the
                             H100 SXM data sheet HBM3 figure; pinned storage reads the frames over PCIe instead)
  sampler_ms_per_batch[net][B]   host sampler (Python `random` replay) per batch
  train[...]                 Wav2LipTrainStep iterations per second at B = 64, T = 5: fed by Wav2LipBatches.next_batch()
                             (sampler + gather in the loop), against the same loop on batches built beforehand; alternated
  reference_loader           a restatement of wav2lip_train.py's __getitem__ (glob, choice, isfile, cv2.imread + cv2.resize
                             of ten frames, load_wav + the full-utterance mel, / 255., transposes, torch.FloatTensor) run on
                             the host with 1 and with 16 processes (as is, and with BLAS and OpenCV held to one thread
                             per process), samples per second.  The mel is oracle/mel_oracle.py
                             (NumPy), standing in for librosa, which the reference uses; label the number as such.
"""
import argparse
import json
import multiprocessing as mp
import os
import random
import subprocess
import sys
import tempfile
import time
from glob import glob
from os.path import basename, dirname, isfile, join

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def make_dataset(root, n_videos, n_frames, seed=0):
    """n_videos videos of n_frames jpg crops (sizes 96..160) and a wav 0.2 s longer than the video, + filelists/train.txt."""
    import cv2
    from scipy.io import wavfile
    from oracle import mel_oracle as M
    rng = np.random.default_rng(seed)
    names = []
    for v in range(n_videos):
        d = join(root, f"v{v:04d}")
        os.makedirs(d, exist_ok=True)
        h, w = (int(x) for x in rng.integers(96, 161, 2))
        base = rng.integers(0, 256, (h, w, 3)).astype(np.int16)
        for f in range(n_frames):
            img = np.clip(base + rng.integers(-12, 13, (h, w, 3)), 0, 255).astype(np.uint8)
            cv2.imwrite(join(d, f"{f}.jpg"), img)
        wav = M.make_wav(int((n_frames / 25. + 0.2) * 16000), seed=v, kind="mix")
        wavfile.write(join(d, "audio.wav"), 16000, (np.clip(wav, -1, 1) * 32767).astype(np.int16))
        names.append(f"v{v:04d}")
    os.makedirs(join(root, "filelists"), exist_ok=True)
    with open(join(root, "filelists", "train.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    return join(root, "filelists", "train.txt")


# ---- a restatement of the reference's per-sample loader (wav2lip_train.py:111-164), for its host throughput ----
def _ref_load_wav(path):
    from scipy.io import wavfile
    _, data = wavfile.read(path)
    return data.astype(np.float32) / np.float32(32768)


def _ref_window(name):
    fid = int(basename(name).split(".")[0])
    paths = [join(dirname(name), f"{i}.jpg") for i in range(fid, fid + 5)]
    return paths if all(isfile(p) for p in paths) else None


def _ref_read(paths):
    import cv2
    out = []
    for p in paths:
        img = cv2.imread(p)
        if img is None:
            return None
        out.append(cv2.resize(img, (96, 96)))
    return out


def _ref_sample(videos, rng):
    import torch
    from oracle import mel_oracle as M
    while True:
        vid = videos[rng.randint(0, len(videos) - 1)]
        names = list(glob(join(vid, "*.jpg")))
        if len(names) <= 15:
            continue
        img, wrong = rng.choice(names), rng.choice(names)
        while wrong == img:
            wrong = rng.choice(names)
        wp, wwp = _ref_window(img), _ref_window(wrong)
        if wp is None or wwp is None:
            continue
        win, wwin = _ref_read(wp), _ref_read(wwp)
        if win is None or wwin is None:
            continue
        spec = M.melspectrogram(_ref_load_wav(join(vid, "audio.wav"))).T
        fid = int(basename(img).split(".")[0])
        s = int(80. * (fid / 25.))
        mel = spec[s:s + 16]
        if mel.shape[0] != 16 or fid < 1:
            continue
        starts = [int(80. * ((i - 2) / 25.)) for i in range(fid + 1, fid + 6)]
        indiv = [spec[k:k + 16] for k in starts]
        if any(m.shape[0] != 16 for m in indiv):
            continue
        window = np.transpose(np.asarray(win) / 255., (3, 0, 1, 2))
        y = window.copy()
        window[:, :, 48:] = 0.
        x = np.concatenate([window, np.transpose(np.asarray(wwin) / 255., (3, 0, 1, 2))], axis=0)
        return (torch.FloatTensor(x), torch.FloatTensor(np.asarray([m.T for m in indiv])).unsqueeze(1),
                torch.FloatTensor(mel.T).unsqueeze(0), torch.FloatTensor(y))


def _ref_worker(args):
    videos, n, seed = args
    import cv2
    import torch
    torch.set_num_threads(1)                       # as DataLoader does in its workers
    if os.environ.get("OPENBLAS_NUM_THREADS") == "1":
        cv2.setNumThreads(1)
    rng = random.Random(seed)
    _ref_sample(videos, rng)                      # imports and first-touch outside the timed window
    t = time.perf_counter()
    for _ in range(n):
        _ref_sample(videos, rng)
    return n, time.perf_counter() - t


def reference_loader(videos, n_per_proc, procs, single_thread=False):
    """Samples per second of `procs` processes (spawned, so that none inherits the parent's CUDA or OpenCV threads), each timing
    its own n_per_proc samples: the sum of the per-process rates.  single_thread: BLAS and OpenCV limited to one thread per
    process (DataLoader limits only torch's)."""
    if procs == 1:
        n, dt = _ref_worker((videos, n_per_proc, 0))
        return n / dt
    keys = ("OPENBLAS_NUM_THREADS", "OMP_NUM_THREADS", "MKL_NUM_THREADS")
    saved = {k: os.environ.get(k) for k in keys}
    if single_thread:
        os.environ.update({k: "1" for k in keys})
    try:
        with mp.get_context("spawn").Pool(procs) as pool:
            return sum(n / dt for n, dt in pool.map(_ref_worker, [(videos, n_per_proc, s) for s in range(procs)]))
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def gather_bytes(net, B):
    if net == "wav2lip":
        return B * (10 * 27648 + 6 * 16 * 80 * 4 + (6 + 3) * 5 * 96 * 96 * 4 + 6 * 80 * 16 * 4)
    return B * (5 * 48 * 96 * 3 + 16 * 80 * 4 + 15 * 48 * 96 * 4 + 80 * 16 * 4 + 4)


def kernel_ms(fn, iters):
    """Mean device time of the gather kernels launched by fn(), from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ts = [getattr(e, "device_time_total", None) or e.cuda_time_total for e in prof.events() if "train_batch_" in e.name]
    ts = [t for t in ts if t > 0]
    return float(np.mean(ts)) / 1e3, len(ts), float(np.min(ts)) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=64)
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--train-iters", type=int, default=30)
    ap.add_argument("--ref-samples", type=int, default=60, help="reference-loader samples per process")
    ap.add_argument("--make-dataset", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.make_dataset:
        print(make_dataset(args.make_dataset, args.videos, args.frames))
        return

    import torch
    from wav2lip_b200 import data as D
    res = {"card": card(), "torch_device": torch.cuda.get_device_name(0), "host_cpus": os.cpu_count(),
           "videos": args.videos, "frames_per_video": args.frames}
    with tempfile.TemporaryDirectory() as tmp:
        flist = make_dataset(tmp, args.videos, args.frames)
        videos = [join(tmp, f"v{v:04d}") for v in range(args.videos)]
        t = time.perf_counter()
        cache = D.TrainDataCache.from_data_root(tmp, "train", filelist=flist)
        res["cache_build_s"] = time.perf_counter() - t
        pinned = D.TrainDataCache(cache.videos, cache.frames.cpu().pin_memory(), cache.mels, cache.device)
        res["gather"] = {}
        res["sampler_ms_per_batch"] = {}
        for net, cls in (("wav2lip", D.Wav2LipBatches), ("syncnet", D.SyncNetBatches)):
            for B in (16, 64):
                b = cls(cache, B, rng=random.Random(1))
                t = time.perf_counter()
                for _ in range(20):
                    table = b.samples(B)
                res["sampler_ms_per_batch"].setdefault(net, {})[B] = (time.perf_counter() - t) / 20 * 1e3
                for storage, c in (("device", cache), ("pinned", pinned)):
                    bb = cls(c, B)
                    ms, n, mn = kernel_ms(lambda: bb.assemble(table), args.iters)
                    nbytes = gather_bytes(net, B)
                    res["gather"].setdefault(storage, {}).setdefault(net, {})[B] = {
                        "kernel_ms": ms, "kernel_ms_min": mn, "launches": n, "bytes": nbytes,
                        "bytes_per_s": nbytes / (ms * 1e-3), "share_of_3.35TB/s": nbytes / (ms * 1e-3) / HBM_BPS}
        # the training step fed by the device pipeline vs pre-built batches (B = 64, T = 5)
        from wav2lip_b200.models import SyncNet_color, Wav2Lip
        from wav2lip_b200.training import Wav2LipTrainStep
        torch.manual_seed(0)
        step = Wav2LipTrainStep(Wav2Lip().cuda().train(), SyncNet_color().cuda().train(), lr=1e-4, syncnet_wt=0.03)
        feed = D.Wav2LipBatches(cache, 64, rng=random.Random(2))
        prebuilt = [feed.next_batch() for _ in range(4)]
        for k in range(3):
            step(*prebuilt[k])
        torch.cuda.synchronize()
        runs = {"fed_by_Wav2LipBatches": [], "prebuilt_batches": []}
        for rep in range(2):
            for mode in ("fed_by_Wav2LipBatches", "prebuilt_batches"):
                torch.cuda.synchronize()
                t = time.perf_counter()
                for i in range(args.train_iters):
                    batch = feed.next_batch() if mode == "fed_by_Wav2LipBatches" else prebuilt[i % 4]
                    step(*batch)
                torch.cuda.synchronize()
                runs[mode].append(args.train_iters / (time.perf_counter() - t))
        res["train_B64_T5_it_per_s"] = runs
        res["reference_loader_oracle_mel_samples_per_s"] = {
            "1_process": reference_loader(videos, args.ref_samples, 1),
            "16_processes": reference_loader(videos, args.ref_samples, 16),
            "16_processes_single_threaded_blas_opencv": reference_loader(videos, args.ref_samples, 16, single_thread=True)}
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
