"""The offline rows of inference.py for the streaming tests — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

One row per output frame: (output index, mel chunk start, video frame index, y1, y2, x1, x2), computed as the reference's
loop computes them on the whole utterance (plain NumPy, restated from the reference):
  chunks        inference.py:231-240, through oracle.pipeline_oracle.mel_chunks on a mel of frame indices
  truncation    inference.py:244  full_frames = full_frames[:len(mel_chunks)]
  boxes         inference.py:87-103 (pad, clip, get_smoothened_boxes :59-66) on the truncated frames' rects, or the
                fixed box of :116-119
  frame of i    inference.py:122  idx = i % len(frames)
"""
import numpy as np

from oracle.pipeline_oracle import mel_chunks


def _get_smoothened_boxes(boxes, T):                      # inference.py:59-66
    for i in range(len(boxes)):
        if i + T > len(boxes):
            window = boxes[len(boxes) - T:]
        else:
            window = boxes[i: i + T]
        boxes[i] = np.mean(window, axis=0)
    return boxes


def _face_detect_boxes(rects, H, W, pads, nosmooth):       # inference.py:87-103 without the detector and the crops
    results = []
    pady1, pady2, padx1, padx2 = pads
    for rect in rects:
        y1 = max(0, rect[1] - pady1)
        y2 = min(H, rect[3] + pady2)
        x1 = max(0, rect[0] - padx1)
        x2 = min(W, rect[2] + padx2)
        results.append([x1, y1, x2, y2])
    boxes = np.array(results)
    if not nosmooth:
        boxes = _get_smoothened_boxes(boxes, T=5)
    return [(y1, y2, x1, x2) for (x1, y1, x2, y2) in boxes]


def offline_rows(n_samples, fps, F, H, W, rects=None, pads=(0, 10, 0, 0), nosmooth=False, box=None):
    n_mel = 1 + n_samples // 200                          # audio.melspectrogram of the whole wav
    if n_mel < 16:
        raise ValueError("shorter than one 16-frame chunk")
    idx = np.arange(n_mel)[None, :]
    starts = [int(c[0, 0]) for c in mel_chunks(idx, fps)]
    n_total = min(len(starts), F)
    if box is not None:
        coords = [tuple(box)] * n_total
    else:
        coords = _face_detect_boxes([tuple(r) for r in np.asarray(rects)[:n_total]], H, W, pads, nosmooth)
    rows = []
    for i, s in enumerate(starts):
        j = i % n_total
        rows.append((i, s, j) + tuple(int(v) for v in coords[j]))
    return np.asarray(rows, dtype=np.int64).reshape(-1, 7)


def random_rects(rng, F, H, W):
    out = []
    for _ in range(F):
        x1, y1 = int(rng.integers(0, W - 20)), int(rng.integers(0, H - 20))
        out.append((x1, y1, int(rng.integers(x1 + 8, W + 3)), int(rng.integers(y1 + 8, H + 3))))
    return np.asarray(out, dtype=np.int64)
