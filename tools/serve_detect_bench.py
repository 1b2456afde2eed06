"""Face detection inside the stream server (DESIGN.md section 3.10).  Not part of bench.py.

25 fps 720p videos of random frames, the generator with random reference-init weights, the detector with the "sparse"
weights of tools/detect_bench.py (make_state_dict(0) with the conf background bias +8: a few hundred candidates per
image, so that every frame has a face) and its loc heads scaled by 1e-3 (boxes near their anchors, inside the frame),
fp16.
  card        name, power limit and max SM clock, read by nvidia-smi in the same run
  ttff        time to the first finished frame of a fresh F = 250 video: detect every frame with
              get_detections_for_batch_u8 (batches of 16) then open(rects=...), against open() with the detector; audio
              given all at once (10 s in one tick), and in real-time 40 ms pieces (a tick every 40 ms of wall time)
  sustained   the most sessions, each in its first pass through a fresh F = 50 video, whose 2 s of audio in 40 ms ticks
              take at most 2 s of wall time (K doubles from 4, then bisects)
  latency     p50 / p90 of tick() host time and of the time from its return to its frames being complete, for 64
              established sessions (rects given) while k fresh detecting sessions tick beside them
  bucket      device time of one S3FD launch of each batch the server uses (1, 4, 16) at 720p, CUDA events around
              w2l_s3fd_detect_u8 on the detector's own context, and the device bytes each plan adds

    python tools/serve_detect_bench.py [--max-sessions 64] [--frames 250] [--out FILE]
    python tools/serve_detect_bench.py --dry-run      (argument parsing and shapes, no GPU)
"""
import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

SR, FPS, PIECE = 16000, 25.0, 640
H, W = 720, 1280
BUCKETS = (1, 4, 16)


def _detector():
    import detect_bench as DB
    from oracle import s3fd_oracle as S
    from wav2lip_b200.face_detection import FaceAlignment, LandmarksType
    from wav2lip_b200.face_detection.detection.sfd.net_s3fd import s3fd
    fa = FaceAlignment(LandmarksType._2D, flip_input=False, device="cuda")
    net = s3fd()
    sd = DB.sparse(S.make_state_dict(0))
    for k in sd:                       # boxes within a few pixels of their anchors: inside the frame
        if "_mbox_loc." in k:
            sd[k] *= 1e-3
    net.load_state_dict(sd, strict=True)
    fa.face_detector.face_detector = net.cuda().eval()
    return fa


def _video(F, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (F, H, W, 3), dtype=torch.uint8, device="cuda", generator=g)


def _audio(seconds, seed=0):
    rng = np.random.default_rng(seed)
    return (0.1 * rng.standard_normal(int(seconds * SR))).astype(np.float32)


def ttff(g, fa, F, mode, pieces):
    """Wall time from having the video and the first audio to the first finished frame on the device."""
    import torch
    from wav2lip_b200.stream import LipSyncServer
    frames = _video(F, seed=F + len(mode) + len(pieces))
    wav = _audio(F / FPS)
    srv = LipSyncServer(g, max_batch=128, detector=fa if mode == "server" else None)
    warm = srv.open(_video(8, seed=1), FPS, box=(100, 356, 400, 624))   # the context, the generator plans
    srv.tick({warm: wav[:16000]}, finish=[warm])
    if mode == "server":   # the detector's weights and plans are built before the clock starts
        w = srv.open(_video(40, seed=2), FPS)
        srv.tick({w: wav[:16000]}, finish=[w])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if mode == "server":
        s = srv.open(frames, FPS)
    else:
        rects = []
        for k in range(0, F, 16):
            rects += fa.get_detections_for_batch_u8(frames[k:k + 16])
        s = srv.open(frames, FPS, rects=[r if r is not None else (500, 200, 760, 480) for r in rects])
    got, i = 0, 0
    e = torch.cuda.Event()
    while not got:
        if pieces == "all":
            out = srv.tick({s: wav}, finish=[s])[s]
        else:
            due = t0 + i * PIECE / SR            # piece i has arrived by then
            while time.perf_counter() < due:
                time.sleep(0.0005)
            out = srv.tick({s: wav[i * PIECE:(i + 1) * PIECE]})[s]
            i += 1
        got = out[1].shape[0]
    e.record()
    e.synchronize()
    dt = time.perf_counter() - t0
    srv.close()
    return {"mode": mode, "audio": pieces, "F": F, "ttff_ms": round(dt * 1e3, 2), "ticks": max(i, 1)}


def sustained(g, fa, K, F=50, seconds=2.0):
    import torch
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(g, max_batch=128, detector=fa)
    w = srv.open(_video(40, seed=3), FPS)                       # plans of the buckets, outside the timed window
    wav = _audio(seconds + 1.0)
    for i in range(30):
        srv.tick({w: wav[i * PIECE:(i + 1) * PIECE]})
    srv.close(w)
    vids = [_video(F, seed=100 + k) for k in range(K)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ids = [srv.open(v, FPS) for v in vids]
    n = int(seconds * SR) // PIECE
    nf = 0
    for i in range(n):
        out = srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in ids})
        nf += sum(v[1].shape[0] for v in out.values() if not isinstance(v, Exception))
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    srv.close()
    return wall <= seconds, wall, nf


def bisect(fn, max_sessions, start=4):
    K, good, bad, trials = start, 0, None, []
    while K <= max_sessions:
        ok, wall, nf = fn(K)
        trials.append({"K": K, "wall_s": round(wall, 4), "frames": nf, "ok": ok})
        if not ok:
            bad = K
            break
        good, K = K, K * 2
    while bad is not None and bad - good > max(1, good // 8):
        K = (good + bad) // 2
        ok, wall, nf = fn(K)
        trials.append({"K": K, "wall_s": round(wall, 4), "frames": nf, "ok": ok})
        good, bad = (K, bad) if ok else (good, K)
    return good, trials


def latency(g, fa, fresh, established=64, ticks=60):
    import torch
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(g, max_batch=128, detector=fa)
    base = _video(250, seed=7)
    rects = [(500, 200, 760, 480)] * 250
    wav = _audio((ticks + 40) * PIECE / SR)
    old = [srv.open(base, FPS, rects=rects) for _ in range(established)]
    for i in range(20):
        srv.tick({s: wav[i * PIECE:(i + 1) * PIECE] for s in old})
    new = [srv.open(_video(250, seed=200 + k), FPS) for k in range(fresh)]
    torch.cuda.synchronize()
    e = torch.cuda.Event()
    host, ready = [], []
    for i in range(20, 20 + ticks):
        piece = wav[i * PIECE:(i + 1) * PIECE]
        t0 = time.perf_counter()
        srv.tick({s: piece for s in old + new})
        t1 = time.perf_counter()
        e.record()
        e.synchronize()
        host.append((t1 - t0) * 1e3)
        ready.append((time.perf_counter() - t1) * 1e3)
    srv.close()
    p = lambda v, q: round(float(np.percentile(v, q)), 3)  # noqa: E731
    return {"established": established, "fresh_detecting": fresh, "tick_host_ms_p50": p(host, 50),
            "tick_host_ms_p90": p(host, 90), "frame_ready_ms_p50": p(ready, 50), "frame_ready_ms_p90": p(ready, 90)}


def bucket(fa, B, iters=10):
    import torch
    net = fa.face_detector.face_detector
    frames = _video(B, seed=300 + B)
    ctx = net._ensure(frames)
    b0 = ctx.device_bytes()
    with torch.no_grad():
        net.detect_u8(frames, 1, reverse_channels=True)
    torch.cuda.synchronize()
    added = ctx.device_bytes() - b0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    with torch.no_grad():
        for _ in range(iters):
            a.record()
            net.detect_u8(frames, 1, reverse_channels=True)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
    return {"bucket": B, "H": H, "W": W, "device_ms": round(float(np.median(ms)), 3),
            "ms_per_frame": round(float(np.median(ms)) / B, 3), "plan_bytes": int(added)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-sessions", type=int, default=64)
    ap.add_argument("--frames", type=int, default=250)
    ap.add_argument("--fresh", default="0,4,8", help="fresh detecting sessions beside the 64 established ones")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--dry-run", action="store_true", help="check the arguments and the sizes, run nothing")
    args = ap.parse_args()
    fresh = [int(v) for v in args.fresh.split(",") if v]
    lines = []

    def emit(r):
        lines.append(r)
        print(json.dumps(r), flush=True)

    if args.dry_run:
        from wav2lip_b200.stream import detect_need
        frame_mb = H * W * 3 / 2 ** 20
        emit({"dry_run": True, "frames": args.frames, "video_MiB": round(args.frames * frame_mb, 1),
              "sustained_video_MiB_at_max": round(args.max_sessions * 50 * frame_mb, 1), "fresh": fresh,
              "buckets": BUCKETS, "frames_open_detects": detect_need(6400, args.frames, H, W, FPS),
              "frames_first_frame_needs": detect_need(6400 + 3200, args.frames, H, W, FPS),
              "audio_samples": int(args.frames / FPS * SR)})
        return
    import serve_bench
    import stream_bench as SB
    emit({"card": serve_bench.card()})
    g = SB._model(True)
    fa = _detector()
    for B in BUCKETS:
        emit({"bucket": bucket(fa, B)})
    for mode in ("rects", "server"):
        for pieces in ("all", "40ms"):
            emit({"ttff": ttff(g, fa, args.frames, mode, pieces)})
    good, trials = bisect(lambda K: sustained(g, fa, K), args.max_sessions)
    emit({"sustained_first_pass_25fps_720p": good, "trials": trials})
    for k in fresh:
        emit({"latency": latency(g, fa, k)})
    emit({"card_after": serve_bench.card()})
    if args.out:
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
