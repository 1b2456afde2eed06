"""preprocess.py's per-frame rules restated in NumPy: which `{i}.jpg` files the script writes for one video, and what each
holds (preprocess.py:38-67 with its abort handling :82-89, face_detection/api.py:64-79).

For frame i of a video, detector batch k = i // batch (`--batch_size`), H x W frames:
  * Box: the detector's top detection d, `np.clip(d, 0, None)` then `int()` of x1, y1, x2, y2: -inf becomes 0, finite
    values truncate toward zero, NaN and +inf raise (ValueError / OverflowError).  No detection: no file.
  * Crop: `fb[j][y1:y2, x1:x2]` clamps the slice ends to H and W; an empty slice makes `cv2.imwrite` raise.
  * Abort: `mp_handler` catches the exception and abandons the rest of the video, keeping the files already written.  A
    non-finite box raises inside get_detections_for_batch, before any file of its batch: the video ends at the start of
    batch k.  An empty crop ends it at frame i.  The earliest point wins.

`rows` is the layout of `w2l_face_crops_u8` (include/w2l.h): (F, 6) int32 of status (0 kept, 1 no face, 2 non-finite box,
3 empty crop, 4 lost after the video's abort), slot (-1 unless kept; kept frames in frame order), y1, y2, x1, x2 (the slice
bounds, a non-finite coordinate leaves 0).  The frame that raised keeps status 2 / 3: the first non-finite box of the
aborting batch, else the empty crop at the abort point.
"""
from __future__ import annotations

import numpy as np

KEPT, NO_FACE, NON_FINITE, EMPTY, ABORTED = 0, 1, 2, 3, 4
NO_ABORT = 2 ** 31 - 1


def frame_box(det, H: int, W: int):
    """get_detections_for_batch's box of one frame and the slice it makes: det is the top detection (>= 4 values, x1 y1 x2
    y2 ...) or None -> (own status, (y1, y2, x1, x2))."""
    if det is None:
        return NO_FACE, (0, 0, 0, 0)
    d = np.clip(np.asarray(det, dtype=np.float32)[:4], 0, None)
    c, status = [0, 0, 0, 0], KEPT
    for k in range(4):
        if np.isnan(d[k]) or np.isinf(d[k]):      # after the clip only NaN and +inf are left
            status = NON_FINITE
        else:
            c[k] = int(d[k])
    x1, y1, x2, y2 = c
    y1, y2, x1, x2 = min(y1, H), min(y2, H), min(x1, W), min(x2, W)   # NumPy slice ends (all >= 0 after the clip)
    if status == KEPT and (y1 >= y2 or x1 >= x2):
        status = EMPTY
    return status, (y1, y2, x1, x2)


def preprocess_rows(dets, H: int, W: int, batch: int = 32) -> np.ndarray:
    """dets: per frame of one video, its top detection or None -> rows (F, 6) int32 as described above."""
    F = len(dets)
    own = [frame_box(d, H, W) for d in dets]
    abort = NO_ABORT
    for i, (s, _) in enumerate(own):
        if s == NON_FINITE:
            abort = min(abort, i - i % batch)
        elif s == EMPTY:
            abort = min(abort, i)
    cause = -1
    if abort < NO_ABORT:
        k = abort // batch
        bad = [i for i in range(k * batch, min(F, (k + 1) * batch)) if own[i][0] == NON_FINITE]
        cause = bad[0] if bad else abort
    rows = np.zeros((F, 6), dtype=np.int32)
    slot = 0
    for i, (s, b) in enumerate(own):
        st = s if (i < abort or i == cause) else ABORTED
        rows[i, 0] = st
        rows[i, 1] = slot if st == KEPT else -1
        slot += st == KEPT
        rows[i, 2:] = b
    return rows


def files(rows: np.ndarray) -> list:
    """The `{i}.jpg` names the script leaves for these rows, in frame order."""
    return ["{}.jpg".format(i) for i in np.flatnonzero(np.asarray(rows)[:, 0] == KEPT)]


def aborted(rows: np.ndarray) -> bool:
    """Whether the video was abandoned (an exception reached mp_handler)."""
    r = np.asarray(rows)[:, 0]
    return bool(np.any((r == NON_FINITE) | (r == EMPTY)))


def crops(frames: np.ndarray, rows: np.ndarray) -> list:
    """The arrays the script hands to cv2.imwrite: frame[y1:y2, x1:x2] of every kept frame, in frame order."""
    return [frames[i][r[2]:r[3], r[4]:r[5]] for i, r in enumerate(np.asarray(rows)) if r[0] == KEPT]
