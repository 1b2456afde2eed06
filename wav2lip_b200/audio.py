"""Mirror of the reference's `audio.melspectrogram` (/root/reference/audio.py:45-51) on the GPU.

`melspectrogram(wav)` keeps the reference's contract — a 1-D float array of 16 kHz samples in,
a float32 (80, 1 + len(wav)//200) array in [-4, 4] out — and additionally accepts a CUDA tensor
(then returns a CUDA tensor and never touches the host).  Constants are hparams.py:33-73; they are
baked into the kernel, there is no `hparams` object to mutate.

`load_wav` / `save_wav` (audio.py:9-15) are host-side file helpers, provided so that the reference's scripts
run unchanged with this module shadowing theirs (inference.py:224 calls `audio.load_wav(path, 16000)`); the
inverse transforms of audio.py are outside the hot path and not provided.  As in the reference (wav2lip_train.py:139-141 runs it inside DataLoader
workers), note that a CUDA-backed function must not be called from forked worker processes.
"""
import ctypes as C
import importlib
import os
import sys

import numpy as np


def _lib():
    try:
        return importlib.import_module("wav2lip_b200._lib")
    except ModuleNotFoundError:
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        if root not in sys.path:
            sys.path.append(root)
        return importlib.import_module("wav2lip_b200._lib")


_ctx = {}


def _context(device: int):
    L = _lib()
    if device not in _ctx:
        _ctx[device] = L.Context(device)
    return _ctx[device]


def load_wav(path, sr):
    """audio.py:9-10 `librosa.core.load(path, sr=sr)[0]`: mono float32 in [-1, 1) at `sr` Hz.
    Uses librosa when it is importable (identical to the reference, resampy kaiser_best included).  Otherwise a
    scipy.io.wavfile reader with librosa's conventions — integer PCM scaled by 2^-(bits-1), channels averaged — and,
    only if the file's rate differs from `sr`, scipy.signal.resample_poly (a polyphase Kaiser FIR: NOT bit-identical to
    resampy's kaiser_best; inference.py:219-221 already makes ffmpeg write 16 kHz files, the common case, where no
    resampling happens and the samples are exact)."""
    try:
        import librosa  # noqa: WPS433
        return librosa.core.load(path, sr=sr)[0]
    except ImportError:
        pass
    from math import gcd

    from scipy.io import wavfile
    rate, data = wavfile.read(path)
    if data.dtype.kind == "i":
        x = data.astype(np.float32) / np.float32(2 ** (8 * data.dtype.itemsize - 1))
    elif data.dtype.kind == "u":  # 8-bit PCM is unsigned, offset 128
        x = (data.astype(np.float32) - 128.0) / 128.0
    else:
        x = data.astype(np.float32)
    if x.ndim > 1:
        x = x.mean(axis=1, dtype=np.float32)
    if sr is not None and int(rate) != int(sr):
        from scipy import signal
        g = gcd(int(rate), int(sr))
        x = signal.resample_poly(x.astype(np.float64), int(sr) // g, int(rate) // g).astype(np.float32)
    return np.ascontiguousarray(x, dtype=np.float32)


def save_wav(wav, path, sr):
    """audio.py:12-15, verbatim semantics (scales `wav` IN PLACE to int16 full scale, as the reference does)."""
    from scipy.io import wavfile
    wav *= 32767 / max(0.01, np.max(np.abs(wav)))
    wavfile.write(path, sr, wav.astype(np.int16))


def num_frames(n_samples: int) -> int:
    return 1 + int(n_samples) // 200


def melspectrogram(wav, device: int = 0):
    L = _lib()
    try:
        import torch
        is_tensor = isinstance(wav, torch.Tensor)
    except ImportError:  # pragma: no cover
        is_tensor = False
    if is_tensor:
        if not wav.is_cuda:
            wav = wav.detach().cpu().numpy()
        else:
            x = wav.detach().contiguous().float().reshape(-1)
            ctx = _context(x.device.index or 0)
            out = torch.empty((80, num_frames(x.numel())), device=x.device, dtype=torch.float32)
            stream = torch.cuda.current_stream(x.device).cuda_stream
            L.check(ctx.lib.w2l_melspectrogram(ctx.h, C.c_void_p(x.data_ptr()), x.numel(), C.c_void_p(out.data_ptr()),
                                               C.c_void_p(stream)))
            return out
    x = np.ascontiguousarray(np.asarray(wav, dtype=np.float32).reshape(-1))
    ctx = _context(device)
    out = np.empty((80, num_frames(x.shape[0])), dtype=np.float32)
    L.check(ctx.lib.w2l_melspectrogram_host(ctx.h, x.ctypes.data_as(C.c_void_p), x.shape[0], out.ctypes.data_as(C.c_void_p)))
    return out


def num_chunks(n_frames: int, fps: float) -> int:
    return int(_lib().get_lib().w2l_mel_num_chunks(int(n_frames), float(fps)))


def mel_chunks(mel, fps: float, device: int = 0):
    """inference.py:231-240 on the GPU: (80,F) mel -> (n_chunks,1,80,16) chunks, one per video frame at `fps`
    (start = int(i*80./fps), last chunk right-aligned) — already the `mel_batch` layout of inference.py:260.
    CUDA tensor in -> CUDA tensor out; numpy in -> numpy out."""
    import torch
    L = _lib()
    is_np = not isinstance(mel, torch.Tensor)
    m = torch.as_tensor(np.ascontiguousarray(mel) if is_np else mel).float()
    if m.dim() != 2 or m.shape[0] != 80:
        raise ValueError(f"expected an (80, F) mel, got {tuple(m.shape)}")
    if not m.is_cuda:
        m = m.cuda(device)
    m = m.contiguous()
    F = m.shape[1]
    n = num_chunks(F, fps)
    if n <= 0:
        raise ValueError(f"mel has {F} frames: shorter than one 16-frame chunk")
    ctx = _context(m.device.index or 0)
    out = torch.empty((n, 1, 80, 16), device=m.device, dtype=torch.float32)
    stream = torch.cuda.current_stream(m.device).cuda_stream
    L.check(ctx.lib.w2l_mel_chunks(ctx.h, C.c_void_p(m.data_ptr()), F, float(fps), C.c_void_p(out.data_ptr()), n,
                                   C.c_void_p(stream)))
    return out.cpu().numpy() if is_np else out


def mel_basis() -> np.ndarray:
    """The kernel's own (80, 401) Slaney filterbank (host computation in libw2l), for inspection."""
    L = _lib()
    out = np.empty((80, 401), dtype=np.float32)
    L.check(L.get_lib().w2l_mel_basis_host(out.ctypes.data_as(C.c_void_p)))
    return out


class MelStream:
    """Streaming `melspectrogram`: push 16 kHz float32 audio as it arrives and get back the mel frames it makes final
    (frame f once 200 f + 400 samples have arrived), each bit-identical to the same column of `melspectrogram` on the
    whole utterance; `finish()` returns the frames that reach the end (1 + L // 200 frames in all).  Device memory is
    two fixed rings (`ring_log2`: log2 of the audio ring in samples, 11..24, default 16), whatever the stream's length.

    `push(pcm)` takes a 1-D numpy array / CPU tensor (returns an (80, k) numpy array) or a CUDA tensor on this stream's
    device (returns an (80, k) CUDA tensor, on the current stream).  `nan_seen()` reports whether any frame so far held
    a NaN (inference.py raises on that)."""

    def __init__(self, device: int = 0, ring_log2: int = 0):
        import torch
        self._torch = torch
        self._ctx = _context(int(device))
        self._lib = self._ctx.lib
        h = C.c_void_p()
        _lib().check(self._lib.w2l_melstream_create(self._ctx.h, int(ring_log2), C.byref(h)))
        self._h = h
        self.device = int(device)
        self._cuda_out = False   # finish() answers in the kind of the pushes
        self._nan_at_finish = None

    def _run(self, pcm, finish: bool):
        torch = self._torch
        L = _lib()
        dev = torch.device("cuda", self.device)
        on_device = isinstance(pcm, torch.Tensor) and pcm.is_cuda
        keep = None
        if pcm is None:
            ptr, n = None, 0
            on_device = self._cuda_out
        elif on_device:
            if pcm.device != dev:
                raise ValueError(f"pcm is on {pcm.device}, the stream on {dev}")
            keep = pcm.detach().reshape(-1).contiguous().float()
            ptr, n = C.c_void_p(keep.data_ptr()), keep.numel()
            self._cuda_out = True
        else:
            x = pcm.detach().cpu().numpy() if isinstance(pcm, torch.Tensor) else pcm
            keep = np.ascontiguousarray(np.asarray(x, dtype=np.float32).reshape(-1))
            ptr, n = keep.ctypes.data_as(C.c_void_p), keep.shape[0]
        k = int(self._lib.w2l_melstream_pending(self._h, n, 1 if finish else 0))
        out = torch.empty((80, k), device=dev, dtype=torch.float32)
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        got = C.c_int64()
        optr = C.c_void_p(out.data_ptr()) if k else None
        if finish:
            flag = C.c_int(0)
            L.check(self._lib.w2l_melstream_finish(self._h, optr, k, C.byref(got), C.byref(flag), stream))
            self._nan_at_finish = bool(flag.value)
        else:
            L.check(self._lib.w2l_melstream_push(self._h, ptr, n, optr, k, C.byref(got), None, stream))
        assert got.value == k
        return out if on_device else out.cpu().numpy()

    def push(self, pcm):
        return self._run(pcm, False)

    def finish(self):
        """The last frames; call once, after the last push.  A CUDA tensor if any push was a CUDA tensor, else numpy."""
        return self._run(None, True)

    def nan_seen(self) -> bool:
        """Whether any frame so far held a NaN (synchronises the current stream)."""
        if self._nan_at_finish is not None:
            return self._nan_at_finish
        torch = self._torch
        flag, got = C.c_int(0), C.c_int64()
        stream = C.c_void_p(torch.cuda.current_stream(torch.device("cuda", self.device)).cuda_stream)
        _lib().check(self._lib.w2l_melstream_push(self._h, None, 0, None, 0, C.byref(got), C.byref(flag), stream))
        return bool(flag.value)

    def close(self):
        if getattr(self, "_h", None):
            self._lib.w2l_melstream_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
