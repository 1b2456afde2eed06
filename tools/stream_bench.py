"""Streaming lip-sync session costs on one GPU (DESIGN.md section 3.8).  Not part of bench.py.

For batch in {1, 4, 16}, with the per-session CUDA graph and without (W2L_DISABLE_STREAMGRAPH=1, read when a context
is created, so each mode gets its own model):
  step_ms      device time of one step on the caller's stream (table copy, gather, crop, generator, paste): CUDA
               events around a push of `batch` frames of audio (one whole step), queued behind a 5 ms sleep kernel so
               that the host has issued the whole push before the device reaches it (no host gap inside the interval;
               the mel work runs on the session's own stream meanwhile)
  span_ms      CUDA events around one push that queues 32 whole steps, per step: the step's device time plus
               whatever gaps the host leaves between steps
  push_ms      host time of push() for 40 ms of audio (one 25 fps output frame)
  ready_ms     time from the return of that push to its frames being complete on the device
and, at batch 1, the number of concurrent 25 fps 720p sessions the GPU sustains: K sessions pushed round-robin in
40 ms pieces for 2 s of audio each, sustained when the whole run takes at most 2 s of wall time; K doubles, then
bisects.  Prints one JSON line per configuration.

    python tools/stream_bench.py [--pushes 200] [--max-sessions 1024]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SR, FPS = 16000, 25.0
PIECE = SR // 25   # 40 ms


def _model(graph: bool):
    os.environ["W2L_DISABLE_STREAMGRAPH"] = "0" if graph else "1"
    from oracle import w2l_oracle as O
    from wav2lip_b200.models import Wav2Lip
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)   # random, reference init
    return g.cuda().eval()


def _video(F, H, W):
    frames = torch.randint(0, 256, (F, H, W, 3), dtype=torch.uint8, device="cuda")
    box = (H // 4, H // 4 + 256, W // 3, W // 3 + 224)
    return frames, box


def _audio(seconds):
    rng = np.random.default_rng(0)
    return (0.1 * rng.standard_normal(int(seconds * SR))).astype(np.float32)


def measure(g, batch, pushes, H=720, W=1280):
    from wav2lip_b200.stream import LipSyncSession
    frames, box = _video(250, H, W)
    wav = _audio((pushes * 2 + 40) * PIECE / SR)
    s = LipSyncSession(g, frames, FPS, box=box, batch=batch)
    at = 0
    for _ in range(20):                     # warm up: plan, graph capture
        s.push(wav[at:at + PIECE]); at += PIECE
    torch.cuda.synchronize()
    # host time of a 40 ms push and the time from its return to its frames being ready
    e = torch.cuda.Event()
    push_ms, ready_ms = [], []
    for _ in range(pushes):
        t0 = time.perf_counter()
        s.push(wav[at:at + PIECE]); at += PIECE
        t1 = time.perf_counter()
        e.record()
        e.synchronize()
        t2 = time.perf_counter()
        push_ms.append((t1 - t0) * 1e3)
        ready_ms.append((t2 - t1) * 1e3)
    # device time of one step: the push is queued behind a sleep kernel, so the events bracket device work only
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    step_ms, late = [], 0
    for _ in range(20):
        torch.cuda.synchronize()
        torch.cuda._sleep(10_000_000)        # ~5 ms at 1.98 GHz
        a.record()
        t0 = time.perf_counter()
        _, fr = s.push(wav[at:at + batch * PIECE]); at += batch * PIECE
        issued = time.perf_counter() - t0
        b.record()
        b.synchronize()
        k = -(-fr.shape[0] // batch)
        if issued > 4e-3:                   # the host was still issuing when the sleep ended: not a clean sample
            late += 1
        elif k:
            step_ms.append(a.elapsed_time(b) / k)
    # span of 32 whole steps queued by one push
    long = _audio(32 * batch * PIECE / SR + 1.0)
    torch.cuda.synchronize()
    a.record()
    _, fr = s.push(long[:32 * batch * PIECE])
    b.record()
    b.synchronize()
    span = a.elapsed_time(b) / max(1, -(-fr.shape[0] // batch))
    s.close()
    med = lambda v: float(np.median(v))  # noqa: E731
    return {"step_ms": med(step_ms) if step_ms else None, "step_samples": len(step_ms), "late": late, "span_ms": span,
            "push_ms": med(push_ms), "push_ms_p90": float(np.percentile(push_ms, 90)),
            "ready_ms": med(ready_ms), "ready_ms_p90": float(np.percentile(ready_ms, 90))}


def sustained(g, K, seconds=2.0, H=720, W=1280):
    """K sessions on one video, round-robin 40 ms pushes on one stream: True if 2 s of audio each takes <= 2 s."""
    from wav2lip_b200.stream import LipSyncSession
    frames, box = _video(250, H, W)
    wav = _audio(seconds + 1.0)
    ss = [LipSyncSession(g, frames, FPS, box=box, batch=1) for _ in range(K)]
    for s in ss:                             # the first 212.5 ms of look-ahead, and the graph capture
        for i in range(8):
            s.push(wav[i * PIECE:(i + 1) * PIECE])
    torch.cuda.synchronize()
    n = int(seconds * SR) // PIECE
    t0 = time.perf_counter()
    frames_out = 0
    for i in range(8, 8 + n):
        for s in ss:
            frames_out += s.push(wav[i * PIECE:(i + 1) * PIECE])[1].shape[0]
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    for s in ss:
        s.close()
    return wall <= seconds, wall, frames_out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pushes", type=int, default=200)
    ap.add_argument("--max-sessions", type=int, default=1024)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    lines = []
    for graph in (True, False):
        g = _model(graph)
        for batch in (1, 4, 16):
            r = {"graph": graph, "batch": batch, **measure(g, batch, args.pushes)}
            lines.append(r)
            print(json.dumps(r), flush=True)
        # concurrent 25 fps 720p sessions at batch 1
        K, good, bad, trials = 8, 0, None, []
        while K <= args.max_sessions:
            ok, wall, nf = sustained(g, K)
            trials.append({"K": K, "wall_s": wall, "frames": nf, "ok": ok})
            if not ok:
                bad = K
                break
            good, K = K, K * 2
        while bad is not None and bad - good > max(1, good // 16):
            K = (good + bad) // 2
            ok, wall, nf = sustained(g, K)
            trials.append({"K": K, "wall_s": wall, "frames": nf, "ok": ok})
            good, bad = (K, bad) if ok else (good, K)
        r = {"graph": graph, "batch": 1, "sessions_25fps_720p": good, "trials": trials}
        lines.append(r)
        print(json.dumps(r), flush=True)
        del g
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
