"""Face detection timing: the host detector path against the device one (`w2l_s3fd_detect_u8`), for B frames of HxW.

    python tools/detect_bench.py [--frames 16] [--height 720] [--width 1280] [--iters 10]

Per weight set it prints one JSON line:
  host_ms            FaceAlignment.get_detections_for_batch on host_frames host uint8 frames (host preprocessing, the
                     network, the 12 maps copied back, NumPy softmax / decode / NMS), wall time ending in a device
                     synchronise; all B frames for "sparse", the first --random-host-frames (1) for "random"
  device_host_in_ms  get_detections_for_batch_u8 on the same host frames (one uint8 H2D copy, then all on the device)
  device_ms          the detector (w2l_s3fd_detect_u8, max_det = 1) on device-resident frames, CUDA events
  network_ms         w2l_s3fd_forward on device-resident fp32 input, CUDA events
  network_conv_ms    sum of the plan's conv launches from profile_plan (cold L2 before each launch)
  select_nms_kernels_ms, u8_ingest_kernel_ms   device time of the post-processing kernels and of the uint8 ingest
                     kernel per detection call (torch.profiler, a separate run)
  candidates         per image, the locations with score > 0.5
Weight sets: "random" = oracle.s3fd_oracle.make_state_dict(0) (random weights: many candidates); "sparse" = the same with
the conf heads' background bias raised by 8, so that only a handful of locations pass, as with a trained detector on
frames with one face.  The card's name and power limit are printed first: the numbers belong to them.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import s3fd_oracle as S  # noqa: E402
from wav2lip_b200.face_detection import FaceAlignment, LandmarksType  # noqa: E402

TAPS = ["conv3_3_norm", "conv4_3_norm", "conv5_3_norm", "fc7", "conv6_2", "conv7_2"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def sparse(sd):
    for i, t in enumerate(TAPS):
        b = sd[f"{t}_mbox_conf.bias"]
        if i == 0:
            b[:3] += 8.0
        else:
            b[0] += 8.0
    return sd


def timed_wall(fn, iters, warmup=True):
    if warmup:
        fn()
        torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def timed_events(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--host-iters", type=int, default=3)
    ap.add_argument("--random-host-frames", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("detect_bench needs a CUDA device")
    print(json.dumps(card()), flush=True)
    B, H, W = args.frames, args.height, args.width
    rgb = S.make_images(B, H, W, seed=0)
    rgb_dev = torch.from_numpy(rgb).cuda()
    x_dev = S.preprocess(np.ascontiguousarray(rgb[..., ::-1])).cuda()
    for name, sd in (("sparse", sparse(S.make_state_dict(0))), ("random", S.make_state_dict(0))):
        fa = FaceAlignment(LandmarksType._2D, flip_input=False, device="cuda")
        net = fa.face_detector.face_detector
        net.load_state_dict(sd, strict=True)
        # with random weights the host path's O(n^2) NMS over ~18 k candidates per 720p image runs for minutes per batch:
        # it is timed once, on the first --random-host-frames frames only (host_frames in the output)
        hf = B if name == "sparse" else min(B, args.random_host_frames)
        fa.get_detections_for_batch(rgb[:1])
        host_ms = timed_wall(lambda: fa.get_detections_for_batch(rgb[:hf]), args.host_iters if name == "sparse" else 1,
                             warmup=False)
        dev_host_ms = timed_wall(lambda: fa.get_detections_for_batch_u8(rgb), args.iters)
        with torch.no_grad():
            dev_ms = timed_events(lambda: net.detect_u8(rgb_dev, 1, reverse_channels=True), args.iters)
            net_ms = timed_events(lambda: net(x_dev), args.iters)
            net.detect_u8(rgb_dev, 1, reverse_channels=True)
        torch.cuda.synchronize()
        ctx = net._w2l_ctx
        cands = [int(n) for n in _counts(ctx, B)]
        conv_ms = sum(ms for _, ms, _ in ctx.profile_plan(3, iters=3))
        post_ms, ingest_ms = kernel_ms(lambda: net.detect_u8(rgb_dev, 1, reverse_channels=True))
        same = fa.get_detections_for_batch_u8(rgb) == fa.get_detections_for_batch(rgb) if name == "sparse" else None
        print(json.dumps({"weights": name, "frames": B, "height": H, "width": W, "host_frames": hf, "host_ms": round(host_ms, 2),
                          "device_host_in_ms": round(dev_host_ms, 3), "device_ms": round(dev_ms, 3),
                          "network_ms": round(net_ms, 3), "network_conv_ms": round(conv_ms, 3),
                          "select_nms_kernels_ms": round(post_ms, 3), "u8_ingest_kernel_ms": round(ingest_ms, 3),
                          "candidates": cands, "same_as_host_path": same}),
              flush=True)


def kernel_ms(fn, iters=5):
    """Device time per call of the select / NMS kernels and of the uint8 ingest kernel, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                fn()
            torch.cuda.synchronize()
    post = ingest = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if any(k in e.key for k in ("s3fd_count_kernel", "s3fd_select_kernel", "s3fd_nms_kernel")):
            post += t
        elif "s3fd_ingest_u8_kernel" in e.key:
            ingest += t
    return post / iters / 1e3, ingest / iters / 1e3


def _counts(ctx, B):
    import ctypes as C
    out = []
    for b in range(B):
        n, path = C.c_int32(), C.c_int32()
        ctx.lib.w2l_debug_s3fd_candidates(ctx.h, b, 0, None, C.byref(n), C.byref(path))
        out.append(n.value)
    return out


if __name__ == "__main__":
    main()
