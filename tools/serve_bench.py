"""Stream group costs on one GPU (DESIGN.md section 3.9).  Not part of bench.py.

25 fps 720p sessions on one random video with a fixed 256 x 224 box, 40 ms pieces, as tools/stream_bench.py does:
  card             name, power limit and max SM clock, read by nvidia-smi in the same run
  sustained        the most sessions whose 2 s of audio each, fed as 40 ms ticks of every session, take at most 2 s of
                   wall time (K doubles from 8, then bisects): for the group at max_batch 64 and 128, and for the
                   per-session baseline (LipSyncSession, batch 1, stream_bench.sustained) in the same run
  latency          at 1, 8 and 64 sessions and at the group's sustained count (max_batch 128): host time of tick() and the
                   time from its return to every frame it returned being complete on the device (p50 / p90)
  step             device time per step for each bucket size: CUDA events around a tick of one whole step, queued behind
                   a sleep kernel so that the host has issued the tick before the device reaches it
  paste            the paste kernel's time and HBM rate (frame bytes read and written / kernel time) from torch.profiler
                   with CUDA activities, in a run of its own, with the time of every kernel of those ticks by name

    python tools/serve_bench.py [--max-sessions 2048] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import stream_bench as SB  # noqa: E402

SR, FPS, PIECE = SB.SR, SB.FPS, SB.PIECE
H, W = 720, 1280


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"name": torch.cuda.get_device_name(), "nvidia_smi": q}


def _server(g, K, max_batch, frames, box):
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(g, max_batch=max_batch)
    ids = [srv.open(frames, FPS, box=box) for _ in range(K)]
    return srv, ids


def sustained_group(g, K, max_batch, seconds=2.0):
    frames, box = SB._video(250, H, W)
    wav = SB._audio(seconds + 1.0)
    srv, ids = _server(g, K, max_batch, frames, box)
    for i in range(8):                       # the first 212.5 ms of look-ahead, plans and graph captures
        srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
    torch.cuda.synchronize()
    n = int(seconds * SR) // PIECE
    t0 = time.perf_counter()
    frames_out = 0
    for i in range(8, 8 + n):
        out = srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
        frames_out += sum(v[1].shape[0] for v in out.values())
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    srv.close()
    return wall <= seconds, wall, frames_out


def bisect(fn, max_sessions, start=8):
    K, good, bad, trials = start, 0, None, []
    while K <= max_sessions:
        ok, wall, nf = fn(K)
        trials.append({"K": K, "wall_s": round(wall, 4), "frames": nf, "ok": ok})
        if not ok:
            bad = K
            break
        good, K = K, K * 2
    while bad is not None and bad - good > max(1, good // 16):
        K = (good + bad) // 2
        ok, wall, nf = fn(K)
        trials.append({"K": K, "wall_s": round(wall, 4), "frames": nf, "ok": ok})
        good, bad = (K, bad) if ok else (good, K)
    return good, trials


def latency(g, K, max_batch=128, ticks=100):
    frames, box = SB._video(250, H, W)
    wav = SB._audio((ticks + 20) * PIECE / SR)
    srv, ids = _server(g, K, max_batch, frames, box)
    for i in range(10):
        srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
    torch.cuda.synchronize()
    e = torch.cuda.Event()
    host, ready = [], []
    for i in range(10, 10 + ticks):
        t0 = time.perf_counter()
        srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
        t1 = time.perf_counter()
        e.record()
        e.synchronize()
        t2 = time.perf_counter()
        host.append((t1 - t0) * 1e3)
        ready.append((t2 - t1) * 1e3)
    srv.close()
    p = lambda v, q: round(float(np.percentile(v, q)), 4)  # noqa: E731
    return {"sessions": K, "tick_host_ms_p50": p(host, 50), "tick_host_ms_p90": p(host, 90),
            "frame_ready_ms_p50": p(ready, 50), "frame_ready_ms_p90": p(ready, 90)}


def step_time(g, B, max_batch=128, samples=10):
    """Device time of one step of bucket B: B sessions whose ticks fix one row each."""
    frames, box = SB._video(250, H, W)
    wav = SB._audio(4.0)
    srv, ids = _server(g, B, max_batch, frames, box)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms, i = [], 0
    while len(ms) < samples and i < 90:
        torch.cuda.synchronize()
        torch.cuda._sleep(10_000_000)        # ~5 ms
        a.record()
        c0 = srv.counters()
        t0 = time.perf_counter()
        out = srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
        issued = time.perf_counter() - t0
        b.record()
        b.synchronize()
        i += 1
        c1 = srv.counters()
        rows = sum(v[1].shape[0] for v in out.values())
        if i > 12 and rows == B and c1[2] - c0[2] == 1 and issued < 4e-3:   # one warm step of exactly B rows
            ms.append(a.elapsed_time(b))
    srv.close()
    return {"bucket": B, "step_ms": round(float(np.median(ms)), 4) if ms else None, "samples": len(ms)}


def paste_profile(g, K, max_batch=128, ticks=20):
    from torch.profiler import ProfilerActivity, profile
    frames, box = SB._video(250, H, W)
    wav = SB._audio((ticks + 20) * PIECE / SR)
    srv, ids = _server(g, K, max_batch, frames, box)
    for i in range(10):
        srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
    torch.cuda.synchronize()
    n_frames = 0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(10, 10 + ticks):
            out = srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
            n_frames += sum(v[1].shape[0] for v in out.values())
        torch.cuda.synchronize()
    srv.close()
    by_name = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            by_name[ev.key] = by_name.get(ev.key, 0.0) + t / 1e3
    paste_ms = sum(v for k, v in by_name.items() if "group_paste_kernel" in k)
    nbytes = 2 * n_frames * H * W * 3
    top = sorted(by_name.items(), key=lambda kv: -kv[1])[:25]
    return {"sessions": K, "ticks": ticks, "frames": n_frames, "paste_ms": round(paste_ms, 4),
            "paste_GBps": round(nbytes / (paste_ms * 1e-3) / 1e9, 1) if paste_ms else None,
            "device_ms_by_kernel": {k[:90]: round(v, 3) for k, v in top}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-sessions", type=int, default=2048)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    lines = []

    def emit(r):
        lines.append(r)
        print(json.dumps(r), flush=True)

    emit({"card": card()})
    g = SB._model(True)
    counts = {}
    for mb in (64, 128):
        good, trials = bisect(lambda K: sustained_group(g, K, mb), args.max_sessions)
        counts[mb] = good
        emit({"group_max_batch": mb, "sessions_25fps_720p": good, "trials": trials})
    good, trials = bisect(lambda K: SB.sustained(g, K), args.max_sessions)
    emit({"baseline_session_batch": 1, "sessions_25fps_720p": good, "trials": trials,
          "group_over_baseline": round(counts[128] / good, 2) if good else None})
    for K in sorted({1, 8, 64, max(1, counts[128])}):
        emit({"latency": latency(g, K)})
    for B in (1, 2, 4, 8, 16, 32, 64, 128):
        emit({"step": step_time(g, B)})
    for K in (64, max(1, counts[128])):
        emit({"profile": paste_profile(g, K)})
    emit({"card_after": card()})
    if args.out:
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
