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
even for frames past the ones a short utterance reaches, which inference.py would not look at.  `LipSyncServer` with a
detector finds the faces itself and removes the second difference for the sessions it detects.
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


class LipSyncServer:
    """Many streaming sessions over one `model`, sharing its context, the caller's stream and the generator steps
    (include/w2l.h `w2l_stream_group_*`, DESIGN.md section 3.9).  Each session gives the same frames as a lone
    `LipSyncSession` fed the same pieces, and as the offline loop, bit for bit.

        srv = LipSyncServer(model, max_batch=128)
        a = srv.open(frames_a, 25.0, rects=rects_a)             # the arguments of LipSyncSession, without batch
        b = srv.open(frames_b, 29.97, box=(y1, y2, x1, x2))
        out = srv.tick({a: pcm_a, b: pcm_b}, finish=[b])       # {session: (first_index, (n, H, W, 3) uint8 CUDA tensor)}
        srv.close(a)

    A tick runs every row its audio fixes, pooled across the sessions it names: full `max_batch` steps, then the rest in
    the smallest power-of-two bucket that holds it.  A session whose audio gives a NaN mel frame fails alone: `tick`
    returns the `ValueError` (the reference's message) as that session's value instead of raising, the other sessions'
    frames are returned as usual, and every later tick that names the failed session raises that `ValueError` before
    anything runs.  A bad argument raises before anything runs, for the whole tick.  `audio_ring_log2` sets the audio
    ring of every session (0: 2^16 samples).

    detector: a `face_detection.FaceAlignment` (as inference.py:69-70 builds it) of the model's precision.  With it,
    `open(frames, fps)` without rects or box finds each frame's face as `get_detections_for_batch_u8` does on
    inference.py's BGR frames, on the device and only for the frames the session's audio reaches, just before a tick
    needs them (DESIGN.md section 3.10); pads and nosmooth apply as with rects.  Its S3FD weights are loaded into the
    model's context and reloaded when they change (rects already found are kept).  A frame that a tick needs without a
    face fails that session as a NaN does, with face_boxes' message naming the frame; a frame the utterance never
    reaches fails nothing."""

    def __init__(self, model, max_batch=128, audio_ring_log2=0, detector=None):
        if isinstance(max_batch, bool) or int(max_batch) != max_batch or int(max_batch) < 1:
            raise ValueError(f"max_batch must be a positive integer, got {max_batch!r}")
        self.model = model
        self.max_batch = int(max_batch)
        self._ring_log2 = int(audio_ring_log2)
        self._h = None
        self._ctx = None
        self._sessions = {}   # id -> (frames, (H, W))
        self._failed = {}     # id -> message
        self.detector = detector
        self._det_loaded = None   # (context, weights key) of the S3FD weights in the model's context
        if detector is not None:
            self._s3fd()

    def _s3fd(self):
        """The detector's S3FD module, checked against the model's precision."""
        net = self.detector.face_detector.face_detector
        if net.precision != self.model.precision:
            raise ValueError(f"the detector's precision ({net.precision}) differs from the model's "
                             f"({self.model.precision}): detection inside the server runs in the model's context")
        return net

    def _group(self, frames):
        ctx = self.model._ensure(frames)   # reloads the weights if the model's parameters changed
        if self._h is None:
            h = C.c_void_p()
            _raise(ctx.lib.w2l_stream_group_create(ctx.h, self.max_batch, self._ring_log2, C.byref(h)))
            self._h, self._ctx, self._lib = h, ctx, ctx.lib
        elif ctx is not self._ctx:
            raise L.W2LError("the model moved to another device or context since the server was created")
        if self.detector is not None:   # the detector's weights, into the model's context, reloaded when they change
            net = self._s3fd()
            key = (ctx, net._weights_key())
            if self._det_loaded is None or self._det_loaded[0] is not key[0] or self._det_loaded[1] != key[1]:
                net._load_into(ctx, torch.cuda.current_stream(frames.device).cuda_stream)
                self._det_loaded = key
        return ctx

    def open(self, frames_u8, fps, rects=None, pads=(0, 10, 0, 0), nosmooth=False, box=None):
        """A new session -> its id (an int)."""
        if not isinstance(frames_u8, torch.Tensor) or not frames_u8.is_cuda:
            raise L.W2LError("frames_u8 must be a CUDA tensor: wav2lip_b200 has no CPU path")
        if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[3] != 3 or frames_u8.shape[0] < 1:
            raise ValueError(f"expected uint8 (F,H,W,3) frames, got {frames_u8.dtype} {tuple(frames_u8.shape)}")
        if not (float(fps) > 0) or not np.isfinite(float(fps)):
            raise ValueError(f"fps must be positive and finite, got {fps!r}")
        detect = rects is None and box is None
        if detect and self.detector is None:
            raise ValueError("pass the detector rects of every frame or one fixed box")
        F, H, W = (int(v) for v in frames_u8.shape[:3])
        desc = _desc(F, H, W, fps, pads, nosmooth, box)
        ra = _rects_array(rects, F) if box is None and not detect else None
        frames = frames_u8.contiguous()
        ctx = self._group(frames)
        self.model._same_device(ctx, frames)
        sid = C.c_int32()
        if detect:
            # the native side orders its first detection after the legacy default stream; frames written on another
            # stream must be complete
            cur = torch.cuda.current_stream(frames.device)
            if cur.cuda_stream != 0:
                cur.synchronize()
            _raise(self._lib.w2l_stream_group_open_detect(self._h, C.c_void_p(frames.data_ptr()), C.byref(desc),
                                                          C.byref(sid)))
        else:
            _raise(self._lib.w2l_stream_group_open(self._h, C.c_void_p(frames.data_ptr()), C.byref(desc),
                                                   ra.ctypes.data_as(C.c_void_p) if ra is not None else None,
                                                   C.byref(sid)))
        self._sessions[sid.value] = (frames, (H, W))
        return sid.value

    def tick(self, pieces, finish=()):
        """pieces: {session: float32 16 kHz samples (host or CUDA), or None}; finish: sessions whose utterance ends
        with this tick (they may be absent from pieces) -> {session: (first_index, frames)} for every session named."""
        if self._h is None:
            raise L.W2LError("no session is open")
        ids = list(pieces.keys()) + [s for s in finish if s not in pieces]
        fin = set(finish)
        for s in ids:
            if s not in self._sessions:
                raise L.W2LError(f"session {s!r} is not open in this server")
            if s in self._failed:
                raise ValueError(self._failed[s])
        frames0 = self._sessions[ids[0]][0] if ids else None
        if frames0 is not None and self._group(frames0) is not self._ctx:
            raise L.W2LError("the model moved to another device or context since the server was created")
        n = len(ids)
        dev = frames0.device if n else None
        keep, ptrs, counts = [], (C.c_void_p * max(n, 1))(), (C.c_int64 * max(n, 1))()
        for i, s in enumerate(ids):
            pcm = pieces.get(s)
            if pcm is None:
                continue
            if isinstance(pcm, torch.Tensor) and pcm.is_cuda:
                if pcm.device != dev:
                    raise ValueError(f"pcm is on {pcm.device}, the server on {dev}")
                k = pcm.detach().reshape(-1).contiguous().float()
                ptrs[i], counts[i] = k.data_ptr(), k.numel()
            else:
                x = pcm.detach().cpu().numpy() if isinstance(pcm, torch.Tensor) else pcm
                k = np.ascontiguousarray(np.asarray(x, dtype=np.float32).reshape(-1))
                ptrs[i], counts[i] = k.ctypes.data, k.shape[0]
            keep.append(k)
        ids_a = (C.c_int32 * max(n, 1))(*ids)
        fin_a = (C.c_int32 * max(n, 1))(*[1 if s in fin else 0 for s in ids])
        need = (C.c_int64 * max(n, 1))()
        _raise(self._lib.w2l_stream_group_pending(self._h, n, ids_a, counts, fin_a, need))
        # one flat output buffer, a view per session
        sizes = [need[i] * self._sessions[s][1][0] * self._sessions[s][1][1] * 3 for i, s in enumerate(ids)]
        flat = torch.empty(max(sum(sizes), 1), device=dev, dtype=torch.uint8) if n else None
        outs, optrs, at = [], (C.c_void_p * max(n, 1))(), 0
        for i, s in enumerate(ids):
            H, W = self._sessions[s][1]
            outs.append(flat[at:at + sizes[i]].view(need[i], H, W, 3))
            optrs[i] = flat.data_ptr() + at if need[i] else None
            at += sizes[i]
        first, got, status = (C.c_int64 * max(n, 1))(), (C.c_int64 * max(n, 1))(), (C.c_int32 * max(n, 1))()
        stream = torch.cuda.current_stream(dev).cuda_stream if n else 0
        _raise(self._lib.w2l_stream_group_tick(self._h, n, ids_a, ptrs, counts, fin_a, optrs, need, first, got, status,
                                               C.c_void_p(stream)))
        res = {}
        for i, s in enumerate(ids):
            if status[i] != L.W2L_OK:
                msg = self._lib.w2l_stream_group_error(self._h, s).decode("utf-8", "replace")
                self._failed[s] = msg
                res[s] = ValueError(msg)
                continue
            assert got[i] == need[i]
            res[s] = (int(first[i]), outs[i])
        if any(got[i] for i in range(n)):
            self.model._range_guard(self._ctx, stream)
        return res

    def counters(self):
        """(CUDA API submissions, host waits, steps) of every tick so far."""
        c, w, st = C.c_int64(), C.c_int64(), C.c_int64()
        if self._h is not None:
            _raise(self._lib.w2l_stream_group_counters(self._h, C.byref(c), C.byref(w), C.byref(st)))
        return c.value, w.value, st.value

    def close(self, session=None):
        """Close one session, or (no argument) the whole server."""
        if session is not None:
            if session not in self._sessions:
                raise L.W2LError(f"session {session!r} is not open in this server")
            _raise(self._lib.w2l_stream_group_close(self._h, session))
            del self._sessions[session]
            self._failed.pop(session, None)
            return
        if self._h is not None:
            self._lib.w2l_stream_group_destroy(self._h)
            self._h = None
        self._sessions.clear()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def detect_need(n_samples, F, H, W, fps, pads=(0, 10, 0, 0), nosmooth=False, final=False):
    """Host only (no GPU): the frames [0, need) whose rects the rows that `n_samples` fix read, as
    `w2l_stream_detect_need` computes them for a detecting session."""
    n = C.c_int64()
    d = _desc(F, H, W, fps, pads, nosmooth, None)
    _raise(L.get_lib().w2l_stream_detect_need(C.byref(d), int(n_samples), 1 if final else 0, C.byref(n)))
    return n.value


def stream_buckets(max_batch, n_rows):
    """Host only (no GPU): the bucket size of each step that `n_rows` pooled rows take in a group of `max_batch`."""
    lib = L.get_lib()
    k = lib.w2l_stream_group_buckets(int(max_batch), int(n_rows), None, 0)
    if k < 0:
        _raise(k)
    out = (C.c_int32 * max(k, 1))()
    lib.w2l_stream_group_buckets(int(max_batch), int(n_rows), out, k)
    return [int(out[i]) for i in range(k)]
