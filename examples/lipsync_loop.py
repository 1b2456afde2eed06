"""The hot loop of the reference's inference.py (:224-271) on the H100 core, with synthetic crops and audio:

    wav --audio.melspectrogram--> mel (80,F) --audio.mel_chunks(fps)--> (n_frames,1,80,16)       inference.py:225, 231-240
    uint8 96x96 BGR crops (what cv2.resize at :126 produces)  +  mel chunks
        --Wav2Lip.infer_stream (batches of N, two in flight)--> uint8 96x96 BGR predictions     inference.py:134-140, 259-269

Everything between the two cv2.resize calls of the reference runs on the GPU; the host only slices batches.

`lipsync_frames` goes one step further (scope row f2): it takes the RAW video frames and face boxes and returns the
finished frames — crop, cv2.resize to 96x96, batch assembly, generator, cv2.resize back to the box and paste
(inference.py:102,:120-140,:259-271), all in one native call per batch (`Wav2Lip.infer_frames`), bit-identical to
OpenCV's fixed-point bilinear resize.
Run:  python examples/lipsync_loop.py [--seconds 20] [--fps 25] [--batch 128] [--frames]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2lip_b200 import audio  # noqa: E402
from wav2lip_b200.models import Wav2Lip  # noqa: E402


def lipsync(model, wav: np.ndarray, crops_u8: np.ndarray, fps: float, batch: int):
    """wav: float32 16 kHz mono; crops_u8: (n_video_frames, 96, 96, 3) uint8 face crops (looped if the audio is longer,
    as inference.py:252 does with its frame list).  Returns (n_audio_frames, 96, 96, 3) uint8 predictions."""
    mel = audio.melspectrogram(torch.from_numpy(wav).cuda())                 # (80, F) on the device
    chunks = audio.mel_chunks(mel, fps).cpu()                                # (n, 1, 80, 16): one chunk per output frame
    n = chunks.shape[0]
    idx = np.arange(n) % len(crops_u8)
    crops = torch.from_numpy(crops_u8)

    def batches():
        for i in range(0, n, batch):
            yield chunks[i:i + batch], crops[idx[i:i + batch]]

    out = torch.empty((n, 96, 96, 3), dtype=torch.uint8)
    i = 0
    for pred in model.infer_stream(batches()):
        out[i:i + pred.shape[0]] = pred
        i += pred.shape[0]
    return out.numpy()


def lipsync_frames(model, wav: np.ndarray, frames_u8: torch.Tensor, boxes, fps: float, batch: int):
    """wav: float32 16 kHz mono; frames_u8: (F,H,W,3) uint8 BGR video frames ON THE DEVICE; boxes: per video frame
    (y1, y2, x1, x2) face boxes (what face_detect returns, inference.py:102).  Returns (n_audio_frames, H, W, 3) uint8
    finished frames on the device: frame i % F with the lip-synced face pasted in (inference.py:120-123, :267-271)."""
    mel = audio.melspectrogram(torch.from_numpy(wav).cuda())
    chunks = audio.mel_chunks(mel, fps)                                      # (n,1,80,16) on the device
    n, F = chunks.shape[0], frames_u8.shape[0]
    out = torch.empty((n,) + tuple(frames_u8.shape[1:]), dtype=torch.uint8, device=frames_u8.device)
    for i in range(0, n, batch):
        idx = np.arange(i, min(i + batch, n)) % F                            # inference.py:121: idx = i % len(frames)
        bx = [[int(f)] + [int(v) for v in boxes[f]] for f in idx]            # rows (frame index, y1, y2, x1, x2)
        out[i:i + len(idx)] = model.infer_frames(chunks[i:i + len(idx)], frames_u8, bx)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", action="store_true", help="start from raw frames + face boxes (crop / resize / paste on the GPU)")
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--fps", type=float, default=25.0)
    ap.add_argument("--batch", type=int, default=128)      # inference.py --wav2lip_batch_size
    ap.add_argument("--checkpoint", default=None, help="a Wav2Lip checkpoint (.pth with 'state_dict'); random weights if omitted")
    args = ap.parse_args()
    model = Wav2Lip()
    if args.checkpoint:
        sd = torch.load(args.checkpoint, map_location="cpu")["state_dict"]
        model.load_state_dict({k.replace("module.", ""): v for k, v in sd.items()})   # inference.py:172-176
    model = model.cuda().eval()
    rng = np.random.RandomState(0)
    wav = (0.1 * rng.randn(int(16000 * args.seconds))).astype(np.float32)
    if args.frames:
        F, H, W = int(args.fps * 4), 360, 640
        frames = torch.from_numpy(rng.randint(0, 256, size=(F, H, W, 3), dtype=np.uint8)).cuda()
        boxes = [(60 + (i % 7), 300 + (i % 5), 200 + (i % 11), 420 + (i % 3)) for i in range(F)]
        lipsync_frames(model, wav, frames, boxes, args.fps, args.batch)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = lipsync_frames(model, wav, frames, boxes, args.fps, args.batch)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        print(f"{out.shape[0]} finished {W}x{H} frames in {dt * 1e3:.1f} ms = {out.shape[0] / dt:.0f} frames/s "
              f"(mel + chunking + crop/resize + generator + resize/paste, all on the device), batch {args.batch}")
        return
    crops = rng.randint(0, 256, size=(int(args.fps * 4), 96, 96, 3), dtype=np.uint8)
    lipsync(model, wav, crops, args.fps, args.batch)       # warm-up with the same batch sizes: an execution plan (buffers,
                                                           # TMA descriptors) is built once per distinct batch size, ~0.1 s each
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = lipsync(model, wav, crops, args.fps, args.batch)
    dt = time.perf_counter() - t0
    print(f"{out.shape[0]} frames ({args.seconds:.0f} s of audio at {args.fps} fps) in {dt * 1e3:.1f} ms "
          f"= {out.shape[0] / dt:.0f} crops/s end to end (mel + chunking + H2D + generator + D2H), batch {args.batch}")


if __name__ == "__main__":
    main()
