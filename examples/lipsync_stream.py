"""Streaming lip-sync: a synthetic face video and synthetic audio pushed in 40 ms pieces, as a TTS engine or a call
would deliver them; every frame comes back as soon as the audio received so far fixes it.  At the end the streamed
frames are checked against the offline loop (`Wav2Lip.infer_frames` on the whole utterance).

    python examples/lipsync_stream.py [--checkpoint wav2lip.pth] [--batch 4]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from wav2lip_b200 import audio  # noqa: E402
from wav2lip_b200.face_detection import face_boxes  # noqa: E402
from wav2lip_b200.models import Wav2Lip  # noqa: E402
from wav2lip_b200.stream import LipSyncSession  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--checkpoint", default=None, help="a reference wav2lip.pth (random weights without)")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--seconds", type=float, default=3.0)
    args = ap.parse_args()

    g = Wav2Lip()
    if args.checkpoint:
        sd = torch.load(args.checkpoint, map_location="cpu")
        g.load_state_dict({k.replace("module.", ""): v for k, v in sd.get("state_dict", sd).items()})
    else:
        from oracle import w2l_oracle as O
        g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
    g = g.cuda().eval()

    # a 2 s, 25 fps, 256 x 320 "video" with a face box that drifts, as a detector would report it
    F, H, W, fps = 50, 256, 320, 25.0
    rng = np.random.default_rng(0)
    frames = torch.from_numpy(rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)).cuda()
    rects = [(80 + i % 7, 60 + i % 5, 200 + i % 3, 190 + i % 4) for i in range(F)]
    t = np.arange(int(args.seconds * 16000)) / 16000.0
    wav = (0.3 * np.sin(2 * np.pi * 180 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t))).astype(np.float32)

    sess = LipSyncSession(g, frames, fps, rects=rects, batch=args.batch)
    out, piece = [], 640                       # 40 ms at 16 kHz
    t0 = time.perf_counter()
    for at in range(0, len(wav), piece):
        first, fr = sess.push(wav[at:at + piece])
        assert first == sum(o.shape[0] for o in out)
        out.append(fr)
    out.append(sess.finish()[1])
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    streamed = torch.cat(out)

    # the offline loop on the whole utterance (inference.py:224-271)
    mel = audio.melspectrogram(wav)
    chunks = torch.from_numpy(audio.mel_chunks(mel, fps)).cuda()
    n_total = min(chunks.shape[0], F)
    boxes = face_boxes(rects[:n_total], H, W)
    rows = np.asarray([(i % n_total,) + tuple(boxes[i % n_total]) for i in range(chunks.shape[0])], dtype=np.int32)
    with torch.no_grad():
        offline = torch.cat([g.infer_frames(chunks[k:k + args.batch], frames, rows[k:k + args.batch])
                             for k in range(0, len(rows), args.batch)])
    same = streamed.shape == offline.shape and torch.equal(streamed, offline)
    print(f"{streamed.shape[0]} frames streamed from {len(wav) / 16000:.2f} s of audio in {dt * 1e3:.1f} ms; "
          f"identical to the offline loop: {same}")
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
