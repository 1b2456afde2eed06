"""Streaming lip-sync: a fixed face video, audio pushed in pieces as it arrives (TTS, a call), finished frames out as
soon as the audio received so far fixes them — the same frames, bit for bit and in the same number, as the offline loop
of inference.py (:224-244 mel and chunks, :87-103 boxes, :120-140 and :259-271 generator and paste) on the whole
utterance.  The rules, and the look-ahead they imply, are in DESIGN.md section 3.8; the native side is
include/w2l.h `w2l_stream_*`.

    sess = LipSyncSession(model, frames_u8, fps, rects=detector_rects)    # or box=(y1, y2, x1, x2)
    for pcm in audio_pieces:               # float32 16 kHz, host or CUDA
        first, frames = sess.push(pcm)     # (n, H, W, 3) uint8 CUDA tensor: output frames first .. first + n - 1
    first, frames = sess.finish()

Two behavioural differences, both in when an error is raised: inference.py raises on a NaN mel before it produces
anything, the session raises the same ValueError from the push that computes the NaN frame (and from every later call),
and frames returned by earlier pushes stay valid; and rects with a None (no face) raise when the session is created,
even for frames past the ones a short utterance reaches, which inference.py would not look at.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L

_NAN_MSG = "Mel contains nan!"


def _desc(F, H, W, fps, pads, nosmooth, box):
    d = L.StreamDesc()
    d.F, d.H, d.W = int(F), int(H), int(W)
    d.fps = float(fps)
    d.nosmooth = 1 if nosmooth else 0
    if box is not None:
        b = [int(v) for v in box]
        if len(b) != 4:
            raise ValueError(f"box must be (y1, y2, x1, x2), got {box!r}")
        d.has_box = 1
        for k in range(4):
            d.box[k] = b[k]
    p = [int(v) for v in pads]
    if len(p) != 4:
        raise ValueError(f"pads must be (top, bottom, left, right), got {pads!r}")
    for k in range(4):
        d.pads[k] = p[k]
    return d


def _rects_array(rects, F):
    if rects is None:
        return None
    if isinstance(rects, torch.Tensor):
        rects = rects.cpu().numpy()
    if not isinstance(rects, np.ndarray):
        rows = list(rects)
        for i, r in enumerate(rows):
            if r is None:  # face_boxes' message (inference.py:91-93)
                raise ValueError(f"Face not detected in frame {i}! Ensure the video contains a face in all the frames.")
        rects = rows
    a = np.ascontiguousarray(np.asarray(rects, dtype=np.int64))
    if a.ndim != 2 or a.shape != (F, 4):
        raise ValueError(f"expected rects of shape ({F}, 4) = (x1, y1, x2, y2) per frame, got {a.shape}")
    if np.abs(a).max(initial=0) >= 2 ** 31:
        raise ValueError("rects out of int32 range")
    return np.ascontiguousarray(a.astype(np.int32))


def _raise(code):
    if code == L.W2L_OK:
        return
    msg = L.get_lib().w2l_last_error().decode("utf-8", "replace")
    if msg.startswith(_NAN_MSG) or "shorter than one 16-frame chunk" in msg:   # as inference.py / audio.mel_chunks
        raise ValueError(msg)
    L.check(code)


def schedule(n_samples, F, H, W, fps, rects=None, pads=(0, 10, 0, 0), nosmooth=False, box=None, final=False,
             first_row=0, cap=None):
    """Host only (no GPU): the rows that `n_samples` received samples fix (all rows of an utterance of that length with
    final=True), as `w2l_stream_schedule` computes them -> (n_fixed, rows) with rows an (n, 7) int32 array of
    (output index, chunk start, frame index, y1, y2, x1, x2) for rows first_row .. first_row + n - 1."""
    lib = L.get_lib()
    d = _desc(F, H, W, fps, pads, nosmooth, box)
    ra = _rects_array(rects, F) if box is None else None
    n_fixed = C.c_int64()
    _raise(lib.w2l_stream_schedule(C.byref(d), ra.ctypes.data_as(C.c_void_p) if ra is not None else None, int(n_samples),
                                   1 if final else 0, 0, 0, None, C.byref(n_fixed)))
    n = max(0, n_fixed.value - int(first_row)) if cap is None else max(0, min(int(cap), n_fixed.value - int(first_row)))
    rows = np.zeros((max(n, 1), L.STREAM_ROW), dtype=np.int32)
    _raise(lib.w2l_stream_schedule(C.byref(d), ra.ctypes.data_as(C.c_void_p) if ra is not None else None, int(n_samples),
                                   1 if final else 0, int(first_row), n, rows.ctypes.data_as(C.c_void_p), C.byref(n_fixed)))
    return n_fixed.value, rows[:n]


class LipSyncSession:
    """One streaming session over `model` (a `wav2lip_b200.models.Wav2Lip` in eval mode, on the device of the frames).

    frames_u8: (F, H, W, 3) uint8 BGR CUDA tensor, the face video (F == 1 for a still image, inference.py --static).
    fps: the video's frame rate (the mel chunk of output i starts at int(i * 80. / fps)).
    rects: F detector rectangles (x1, y1, x2, y2), as `FaceAlignment.get_detections_for_batch_u8` returns them, padded
        by `pads` (top, bottom, left, right) and smoothed over 5 frames unless `nosmooth`; or
    box: one fixed (y1, y2, x1, x2) box for every frame (inference.py --box).
    batch: rows per generator step.  Each push runs ceil(ready / batch) steps of exactly `batch` rows.
    Weights reloaded into `model` between pushes are picked up by the next push."""

    def __init__(self, model, frames_u8, fps, rects=None, pads=(0, 10, 0, 0), nosmooth=False, box=None, batch=1):
        if not isinstance(frames_u8, torch.Tensor) or not frames_u8.is_cuda:
            raise L.W2LError("frames_u8 must be a CUDA tensor: wav2lip_b200 has no CPU path")
        if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[3] != 3 or frames_u8.shape[0] < 1:
            raise ValueError(f"expected uint8 (F,H,W,3) frames, got {frames_u8.dtype} {tuple(frames_u8.shape)}")
        if isinstance(batch, bool) or int(batch) != batch or int(batch) < 1:
            raise ValueError(f"batch must be a positive integer, got {batch!r}")
        if not (float(fps) > 0) or not np.isfinite(float(fps)):
            raise ValueError(f"fps must be positive and finite, got {fps!r}")
        if rects is None and box is None:
            raise ValueError("pass the detector rects of every frame or one fixed box")
        F, H, W = (int(v) for v in frames_u8.shape[:3])
        self._desc = _desc(F, H, W, fps, pads, nosmooth, box)
        self._rects = _rects_array(rects, F) if box is None else None
        self.model = model
        self.frames = frames_u8.contiguous()
        self.shape = (H, W)
        ctx = model._ensure(self.frames)
        model._same_device(ctx, self.frames)
        self._ctx = ctx
        self._lib = ctx.lib
        h = C.c_void_p()
        _raise(self._lib.w2l_stream_create(ctx.h, C.c_void_p(self.frames.data_ptr()), C.byref(self._desc),
                                           self._rects.ctypes.data_as(C.c_void_p) if self._rects is not None else None,
                                           int(batch), C.byref(h)))
        self._h = h
        self.batch = int(batch)

    def _call(self, pcm, finish):
        if not getattr(self, "_h", None):
            raise L.W2LError("the session is closed")
        ctx = self.model._ensure(self.frames)   # reloads the weights if the model's parameters changed
        if ctx is not self._ctx:
            raise L.W2LError("the model moved to another device or context since the session was created")
        dev = self.frames.device
        keep, ptr, n = None, None, 0
        if pcm is not None:
            if isinstance(pcm, torch.Tensor) and pcm.is_cuda:
                if pcm.device != dev:
                    raise ValueError(f"pcm is on {pcm.device}, the session on {dev}")
                keep = pcm.detach().reshape(-1).contiguous().float()
                ptr, n = C.c_void_p(keep.data_ptr()), keep.numel()
            else:
                x = pcm.detach().cpu().numpy() if isinstance(pcm, torch.Tensor) else pcm
                keep = np.ascontiguousarray(np.asarray(x, dtype=np.float32).reshape(-1))
                ptr, n = keep.ctypes.data_as(C.c_void_p), keep.shape[0]
        need = C.c_int64()
        _raise(self._lib.w2l_stream_pending(self._h, n, 1 if finish else 0, C.byref(need)))
        out = torch.empty((need.value,) + self.shape + (3,), device=dev, dtype=torch.uint8)
        stream = torch.cuda.current_stream(dev).cuda_stream
        first, got = C.c_int64(), C.c_int64()
        optr = C.c_void_p(out.data_ptr()) if need.value else None
        if finish:
            _raise(self._lib.w2l_stream_finish(self._h, optr, need.value, C.byref(first), C.byref(got), C.c_void_p(stream)))
        else:
            _raise(self._lib.w2l_stream_push(self._h, ptr, n, optr, need.value, C.byref(first), C.byref(got),
                                             C.c_void_p(stream)))
        assert got.value == need.value
        if got.value:
            self.model._range_guard(ctx, stream)
        return int(first.value), out

    def push(self, pcm):
        """Append float32 16 kHz samples -> (first_index, (n, H, W, 3) uint8 CUDA tensor) of the frames they fix."""
        return self._call(pcm, False)

    def finish(self):
        """End of the utterance -> (first_index, the remaining frames)."""
        return self._call(None, True)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.w2l_stream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
