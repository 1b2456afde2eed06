"""preprocess.py + the training cache, on synthetic seeded videos: the device path against the reference-shaped one.

    python tools/preprocess_bench.py [--videos 64] [--frames 100] [--hd-videos 8] [--repeats 3]

Two sets: --videos videos of --frames frames at 160x160 (the LRS2 face-track size), and --hd-videos videos of --frames
frames at 1280x720.  Frames are seeded uint8 noise in host memory, each video has 16 kHz audio of its length.  The detector
is oracle.s3fd_oracle.make_state_dict(0) with the conf heads' background bias raised by 8 ("sparse": a few hundred
locations pass per 720p image, as with a trained detector on frames with one face).  Per set it prints one JSON line:
  from_videos_fps      frames per second of TrainDataCache.from_videos from host frames (detector, face_crops, device mel),
                       wall time ending in the device synchronise _build makes; median of --repeats after one warm-up
  reference_fps        frames per second of the reference-shaped path on the same GPU: get_detections_for_batch_u8 per 32
                       frames, cv2.imwrite of each crop ({i}.jpg, as preprocess.py writes them) and the audio.wav, then
                       TrainDataCache.from_data_root (decode on 16 threads, device resize, device mel); median of --repeats
  kernels_us           face_crops_rows_kernel / face_crops_resize_kernel device time per launch, torch.profiler over one
                       from_videos call in a separate run, with the launch count and the kept frames
The card's name, power limit and max SM clock are printed first: the numbers belong to them.  Files go to a temporary
directory that is removed at the end.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import s3fd_oracle as S  # noqa: E402
from wav2lip_b200 import data as D  # noqa: E402
from wav2lip_b200.face_detection import FaceAlignment, LandmarksType  # noqa: E402
from wav2lip_b200.face_detection.detection.sfd.net_s3fd import s3fd  # noqa: E402

TAPS = ["conv3_3_norm", "conv4_3_norm", "conv5_3_norm", "fc7", "conv6_2", "conv7_2"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def detector():
    sd = S.make_state_dict(0)
    for i, t in enumerate(TAPS):
        b = sd[f"{t}_mbox_conf.bias"]
        if i == 0:
            b[:3] += 8.0
        else:
            b[0] += 8.0
    fa = FaceAlignment(LandmarksType._2D, flip_input=False, device="cuda")
    m = s3fd()
    m.load_state_dict(sd, strict=True)
    fa.face_detector.face_detector = m.cuda().eval()
    return fa


def make_videos(n, F, H, W, seed):
    rng = np.random.default_rng(seed)
    return [{"path": f"set/vid{i:03d}", "frames": rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8),
             "wav": (rng.standard_normal(F * 640) * 0.1).astype(np.float32), "sr": 16000} for i in range(n)]


def run_device(fa, videos):
    t = time.perf_counter()
    cache = D.TrainDataCache.from_videos(iter(videos), fa)
    return time.perf_counter() - t, cache.n_frames


def run_reference(fa, videos, root):
    """preprocess.py's loop with the device detector, then the Dataset-side cache from its files."""
    import cv2
    from scipy.io import wavfile
    import shutil
    shutil.rmtree(root, ignore_errors=True)
    t = time.perf_counter()
    names = []
    for v in videos:
        fulldir = os.path.join(root, v["path"])
        os.makedirs(fulldir, exist_ok=True)
        frames = v["frames"]
        try:
            i = -1
            for s in range(0, len(frames), 32):
                fb = frames[s:s + 32]
                for j, f in enumerate(fa.get_detections_for_batch_u8(fb)):
                    i += 1
                    if f is None:
                        continue
                    x1, y1, x2, y2 = f
                    if not cv2.imwrite(os.path.join(fulldir, "{}.jpg".format(i)), fb[j][y1:y2, x1:x2]):
                        raise OSError("imwrite")
        except Exception:  # noqa: BLE001  (mp_handler abandons the video)
            pass
        wavfile.write(os.path.join(fulldir, "audio.wav"), 16000, (np.clip(v["wav"], -1, 1) * 32767).astype(np.int16))
        names.append(v["path"])
    flist = os.path.join(root, "train.txt")
    with open(flist, "w") as f:
        f.write("\n".join(names) + "\n")
    cache = D.TrainDataCache.from_data_root(root, "train", filelist=flist)
    return time.perf_counter() - t, cache.n_frames


def kernel_times(fa, videos):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cache = D.TrainDataCache.from_videos(iter(videos), fa)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("face_crops_rows_kernel", "face_crops_resize_kernel"):
            if k in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                out[k] = {"us_per_launch": round(t / max(1, e.count), 2), "launches": e.count}
    out["kept_frames"] = cache.n_frames
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=64)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--hd-videos", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "preprocess_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    fa = detector()
    with tempfile.TemporaryDirectory() as tmp:
        for name, n, H, W in (("160x160", a.videos, 160, 160), ("1280x720", a.hd_videos, 720, 1280)):
            videos = make_videos(n, a.frames, H, W, seed=H)
            total = n * a.frames
            run_device(fa, videos[:1])            # plans, pinned blocks, library load
            run_reference(fa, videos[:1], os.path.join(tmp, "warm"))
            dev, ref = [], []
            for _ in range(a.repeats):           # alternated
                dev.append(run_device(fa, videos))
                ref.append(run_reference(fa, videos, os.path.join(tmp, name)))
            kt = kernel_times(fa, videos)
            res = {"set": name, "videos": n, "frames_per_video": a.frames, "frames": total,
                   "kept_device": dev[0][1], "kept_reference": ref[0][1],
                   "from_videos_s": [round(t, 3) for t, _ in dev], "reference_s": [round(t, 3) for t, _ in ref],
                   "from_videos_fps": round(total / float(np.median([t for t, _ in dev])), 1),
                   "reference_fps": round(total / float(np.median([t for t, _ in ref])), 1),
                   "launch_frames": D._launch_frames(H, W, 32), "kernels_us": kt}
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
