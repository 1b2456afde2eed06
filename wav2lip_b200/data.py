"""The training scripts' data pipeline on the GPU: a device cache of the preprocessed dataset and batch assembly in one launch.

The reference's `Dataset.__getitem__` (wav2lip_train.py:111-164, identical in hq_wav2lip_train.py; color_syncnet_train.py:69-131)
re-reads ten jpgs, re-resizes them and recomputes the whole utterance's mel for every sample on the CPU.  Here:

  cache = TrainDataCache.from_data_root(data_root, "train")      # once per run: decode, resize, mel
  for x, indiv_mels, mel, gt in Wav2LipBatches(cache, 16).epoch():  # = DataLoader(Dataset("train"), batch_size=16)
      ...

* `TrainDataCache` holds every `*.jpg` as `cv2.resize(cv2.imread(f), (96, 96))` in one uint8 (n, 96, 96, 3) BGR tensor (on the
  device, or in pinned host memory for datasets larger than HBM), resized on the device by the `cv2.resize`-exact
  `w2l_crop_resize_u8`, and every video's `orig_mel = audio.melspectrogram(wav).T` computed once on the device.  The host index
  keeps each video's jpg names in the order `glob` returned them when the cache was built, which frames were unreadable and
  whether the audio failed.
* `Wav2LipBatches` / `SyncNetBatches` replay the reference's `random` draws call for call on that index (the same rejection rules,
  reading the cache's flags instead of the files), then one gather kernel (`w2l_train_batch_wav2lip` / `_syncnet`) writes what
  `default_collate` of B `__getitem__` calls holds.  With the same glob order, `random.seed(s)` and `num_workers=0`, the batches
  are bit-identical to the reference's for x, gt and y, and for the mel windows given the same `orig_mel`.  The device mel is
  within 1e-4 of the reference's (and differs where `load_wav` resamples, see audio.py).  With forked DataLoader workers the
  reference's draw order depends on torch's per-worker seeds; that order is not reproduced, only the sampling distribution.

Host decode (`scan_data_root`, `decode_video`) is separate from the device part.  There is no CPU fallback for the latter.

preprocess.py itself (the step that makes the jpgs) also runs on the device, from decoded videos:

  cache = TrainDataCache.from_videos(({"path": p, "frames": f, "wav": w, "sr": sr} for ...), FaceAlignment(...))

* `face_crops` is preprocess.py's `process_video_file` (:38-67, with mp_handler's abort rules :82-89) for one video: the S3FD
  detector (`w2l_s3fd_detect_u8`) and `w2l_face_crops_u8` leave a row per frame (kept / no face / non-finite box / empty crop /
  lost after the video's abort, and the slice bounds) and `cv2.resize(frame[y1:y2, x1:x2], (96, 96))` of every kept frame on
  the device, with no host sync until the rows are read.  `from_videos` builds the cache from them, names `{i}.jpg` as the
  script's files.  Deliberate deviation: the cache holds the resize of the raw crop, where the reference's training data went
  through a JPEG round trip (`cv2.imwrite`, then `cv2.imread` in the Dataset).  `write_face_crops` writes the script's files
  byte for byte from the same rows instead, for the reference's own scripts or `from_data_root`.
"""
from __future__ import annotations

import ctypes as C
import os
import random as _random
from concurrent.futures import ThreadPoolExecutor
from glob import glob
from os.path import basename, join

import numpy as np

SYNCNET_T = 5            # wav2lip_train.py:36
MEL_STEP = 16            # syncnet_mel_step_size
FPS = 25                 # hparams.fps
IMG = 96                 # hparams.img_size
SAMPLE_RATE = 16000      # hparams.sample_rate
W2L_FIELDS, SYNC_FIELDS = 17, 8   # sample-row widths of include/w2l.h w2l_train_batch_wav2lip / _syncnet
_CANVAS_BYTES = 64 << 20          # host canvas per resize launch
_LAUNCH_PIXELS = 1 << 22          # frame pixels per detector launch of face_crops (DESIGN.md section 3.12)


def get_image_list(data_root: str, split: str, filelist: str = None) -> list:
    """hparams.get_image_list: `filelists/{split}.txt` relative to the current directory (or `filelist`), first word of each
    line joined to `data_root`."""
    out = []
    with open(filelist if filelist is not None else "filelists/{}.txt".format(split)) as f:
        for line in f:
            line = line.strip()
            if " " in line:
                line = line.split()[0]
            out.append(os.path.join(data_root, line))
    return out


def scan_data_root(data_root: str, split: str, filelist: str = None) -> list:
    """[(video dir, [jpg basenames in glob order])] for every video of the split (wav2lip_train.py:42, :115)."""
    return [(vid, [basename(p) for p in glob(join(vid, "*.jpg"))]) for vid in get_image_list(data_root, split, filelist)]


def _imread(path):
    import cv2
    img = cv2.imread(path)
    # read_window (wav2lip_train.py:63-70) rejects a frame that imread cannot decode or cv2.resize refuses
    return img if img is not None and img.ndim == 3 and img.shape[2] == 3 and img.size > 0 else None


def decode_video(vid: str, img_names: list, pool: ThreadPoolExecutor = None) -> dict:
    """Host half of one video: {"img_names", "crops": [uint8 (h, w, 3) BGR or None if unreadable], "wav": float32 or None if
    `audio.load_wav(join(vid, "audio.wav"), 16000)` raised}."""
    from . import audio
    paths = [join(vid, n) for n in img_names]
    crops = list(pool.map(_imread, paths)) if pool is not None else [_imread(p) for p in paths]
    try:
        wav = audio.load_wav(join(vid, "audio.wav"), SAMPLE_RATE)
    except Exception:
        wav = None
    return {"path": vid, "img_names": img_names, "crops": crops, "wav": wav}


def _cache_device(storage, device):
    import torch
    if storage not in ("device", "pinned"):
        raise ValueError(f"storage must be 'device' or 'pinned', got {storage!r}")
    return torch.device("cuda", torch.cuda.current_device() if device is None else torch.device(device).index or 0)


def _launch_frames(H: int, W: int, batch_size: int) -> int:
    """Frames per detector launch in `face_crops`: batch_size * 2^k, the most that stay within _LAUNCH_PIXELS frame pixels
    (at least batch_size), so that every launch starts at a multiple of batch_size and a frame size has one S3FD plan."""
    n = batch_size
    while 2 * n * H * W <= _LAUNCH_PIXELS:
        n *= 2
    return n


def face_crops(detector, frames, batch_size: int = 32, out=None):
    """preprocess.py's `process_video_file` (:38-67) for one video on the device, up to the jpgs: frames (F,H,W,3) uint8 BGR
    (host memory or a CUDA tensor), `detector` this package's `face_detection.FaceAlignment`, `batch_size` the script's
    --batch_size, which only sets where a non-finite box ends the video (mp_handler, :82-89).
    -> rows (F, 6) int32 ndarray, one per frame: status (0 kept, 1 no face, 2 non-finite box, 3 empty crop, 4 lost after the
       video's abort), slot (-1 unless kept), y1, y2, x1, x2 (include/w2l.h w2l_face_crops_u8; oracle/preprocess_oracle.py);
       crops (n_kept, 96, 96, 3) uint8 = cv2.resize(frame[y1:y2, x1:x2], (96, 96)) of the kept frames in frame order, in
       `out` (uint8 (cap, 96, 96, 3), device or pinned host memory; default: a new device tensor of F slots).
    The detector sees each frame as get_detections_for_batch does (channels reversed), in launches sized from H x W (the top
    box of an image does not depend on its batch, DESIGN.md section 3.6), the last one padded.  Host frames are staged
    through pinned memory.  The host waits only once, for the rows, at the end."""
    import torch
    from . import _lib
    if isinstance(batch_size, bool) or int(batch_size) != batch_size or batch_size < 1:
        raise ValueError(f"batch_size must be a positive int, got {batch_size!r}")
    batch_size = int(batch_size)
    net = detector.face_detector.face_detector           # FaceAlignment -> SFDDetector -> the s3fd module
    dev = next(net.parameters()).device
    if dev.type != "cuda":
        raise ValueError("the detector must be on a CUDA device")
    x = frames if isinstance(frames, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(frames)))
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3:
        raise ValueError(f"expected (F,H,W,3) uint8 frames, got {x.dtype} {tuple(x.shape)}")
    if x.is_cuda and x.device != dev:
        raise ValueError(f"frames are on {x.device}, the detector on {dev}")
    x = x.contiguous()
    F, H, W, _ = x.shape
    if out is None:
        out = torch.empty((F, IMG, IMG, 3), dtype=torch.uint8, device=dev)
    elif not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or tuple(out.shape[1:]) != (IMG, IMG, 3) \
            or not out.is_contiguous() or not (out.device == dev or (not out.is_cuda and out.is_pinned())):
        raise ValueError(f"out must be a contiguous uint8 (cap, 96, 96, 3) tensor on {dev} or in pinned host memory")
    rows = torch.empty((F, 6), dtype=torch.int32, device=dev)
    if F == 0:
        return rows.cpu().numpy(), out[:0]
    L = _launch_frames(H, W, batch_size)
    state = torch.zeros((2,), dtype=torch.int32, device=dev)
    pad = None
    stream = torch.cuda.current_stream(dev)

    def p(t):
        return C.c_void_p(t.data_ptr())
    with torch.no_grad(), torch.cuda.device(dev):
        for s in range(0, F, L):
            n = min(L, F - s)
            if x.is_cuda and n == L:
                src = x[s:s + L]
            else:
                if pad is None:
                    pad = torch.zeros((L, H, W, 3), dtype=torch.uint8, device=dev)
                if x.is_cuda:
                    pad[:n].copy_(x[s:s + n])
                else:   # a fresh block of the caching host allocator, reused once its copy has completed
                    stage = torch.empty((n, H, W, 3), dtype=torch.uint8, pin_memory=True)
                    stage.copy_(x[s:s + n])
                    pad[:n].copy_(stage, non_blocking=True)
                src = pad
            dets, counts, _ = net.detect_u8(src, 1, reverse_channels=True)
            ctx = net._w2l_ctx
            _lib.check(ctx.lib.w2l_face_crops_u8(ctx.h, p(src), n, H, W, p(dets), p(counts), 1, s, batch_size, p(state),
                                                 p(rows[s:]), p(out), out.shape[0], C.c_void_p(stream.cuda_stream)))
    st = state.cpu().numpy()
    rows = rows.cpu().numpy()
    if int(st[0]) > out.shape[0]:
        raise ValueError(f"{int(st[0])} kept frames do not fit the {out.shape[0]} slots of out")
    return rows, out[:int(st[0])]


def write_face_crops(fulldir: str, frames, rows) -> list:
    """preprocess.py's files from `face_crops`' rows, on the host: cv2.imwrite(join(fulldir, "{i}.jpg"), frame[y1:y2, x1:x2])
    for every kept frame i (preprocess.py:67), byte-identical to the script's for the same boxes.  -> the names written."""
    import cv2
    os.makedirs(fulldir, exist_ok=True)
    if hasattr(frames, "cpu"):
        frames = frames.cpu().numpy()
    names = []
    for i, r in enumerate(np.asarray(rows)):
        if r[0] == 0:
            names.append("{}.jpg".format(i))
            if not cv2.imwrite(join(fulldir, names[-1]), frames[i][r[2]:r[3], r[4]:r[5]]):
                raise OSError(f"cv2.imwrite failed for {join(fulldir, names[-1])}")
    return names


class VideoIndex:
    """Host index of one cached video: jpg names in glob order, name -> frame slot (-1: unreadable), and its mel rows
    [mel_off, mel_off + mel_len) in the cache (mel_len -1: the audio failed)."""
    __slots__ = ("path", "img_names", "slots", "mel_off", "mel_len")

    def __init__(self, path, img_names, slots, mel_off, mel_len):
        self.path, self.img_names, self.mel_off, self.mel_len = path, list(img_names), int(mel_off), int(mel_len)
        self.slots = dict(zip(self.img_names, (int(s) for s in slots)))


def _frame_id(name: str) -> int:
    return int(basename(name).split(".")[0])          # get_frame_id


def _mel_start(frame_num: int) -> int:
    return int(80. * (frame_num / float(FPS)))        # crop_audio_window


def _window(v: VideoIndex, name: str):
    """get_window + read_window: the 5 slots of ids id..id+4, or None if one is missing or unreadable."""
    start = _frame_id(name)
    out = []
    for fid in range(start, start + SYNCNET_T):
        s = v.slots.get("{}.jpg".format(fid), -1)
        if s < 0:
            return None
        out.append(s)
    return out


def _mel_row(v: VideoIndex, frame_num: int):
    """Absolute cache row of the mel window at frame_num, or None where `spec[start:start+16]` is shorter than 16 rows."""
    r = _mel_start(frame_num)
    return v.mel_off + r if r + MEL_STEP <= v.mel_len else None


def sample_wav2lip(videos: list, rng=_random) -> list:
    """One wav2lip_train.py `__getitem__` (:111-164) on the index: the same `rng` calls in the same order and the same rejections.
    -> [window slots x5, wrong-window slots x5, mel row, indiv rows x5, video end row]."""
    while 1:
        v = videos[rng.randint(0, len(videos) - 1)]
        names = v.img_names
        if len(names) <= 3 * SYNCNET_T:
            continue
        img_name = rng.choice(names)
        wrong_img_name = rng.choice(names)
        while wrong_img_name == img_name:
            wrong_img_name = rng.choice(names)
        window, wrong = _window(v, img_name), _window(v, wrong_img_name)
        if window is None or wrong is None or v.mel_len < 0:
            continue
        fid = _frame_id(img_name)
        mel = _mel_row(v, fid)
        if mel is None:
            continue
        if fid + 1 - 2 < 0:                            # get_segmented_mels: start_frame_num - 2 < 0
            continue
        indiv = [_mel_row(v, i - 2) for i in range(fid + 1, fid + 1 + SYNCNET_T)]
        if any(r is None for r in indiv):
            continue
        return window + wrong + [mel] + indiv + [v.mel_off + v.mel_len]


def sample_syncnet(videos: list, rng=_random) -> list:
    """One color_syncnet_train.py `__getitem__` (:69-131) on the index -> [window slots x5, mel row, label, video end row].
    The mel is cut at img_name even when y = 0 took the frames from wrong_img_name (:118)."""
    while 1:
        v = videos[rng.randint(0, len(videos) - 1)]
        names = v.img_names
        if len(names) <= 3 * SYNCNET_T:
            continue
        img_name = rng.choice(names)
        wrong_img_name = rng.choice(names)
        while wrong_img_name == img_name:
            wrong_img_name = rng.choice(names)
        if rng.choice([True, False]):
            y, chosen = 1, img_name
        else:
            y, chosen = 0, wrong_img_name
        window = _window(v, chosen)
        if window is None or v.mel_len < 0:
            continue
        mel = _mel_row(v, _frame_id(img_name))
        if mel is None:
            continue
        return window + [mel, y, v.mel_off + v.mel_len]


class TrainDataCache:
    """The dataset on the GPU: `frames` uint8 (n, 96, 96, 3) BGR (device, or pinned host memory), `mels` fp32 (rows, 80) on
    the device, `videos` the host index (list of VideoIndex, in filelist order)."""

    def __init__(self, videos, frames, mels, device):
        self.videos, self.frames, self.mels, self.device = videos, frames, mels, device

    @classmethod
    def from_data_root(cls, data_root: str, split: str, filelist: str = None, storage: str = "device", device=None,
                       workers: int = 16) -> "TrainDataCache":
        """Scan `data_root` as the reference's Dataset(split) does (hparams.get_image_list quirk included: `filelists/{split}.txt`
        is opened relative to the current directory unless `filelist` is given), decode with cv2 on `workers` threads."""
        scan = scan_data_root(data_root, split, filelist)
        with ThreadPoolExecutor(max(1, int(workers))) as pool:
            return cls._build(scan, (decode_video(vid, names, pool) for vid, names in scan), storage, device)

    @classmethod
    def from_arrays(cls, videos, storage: str = "device", device=None) -> "TrainDataCache":
        """videos: one dict per video with "img_names" (glob order), "crops" (uint8 (h, w, 3) BGR of any size, None = unreadable)
        and either "wav" (float 16 kHz samples) or "mel" (`orig_mel`, (rows, 80)); a missing / None audio = the audio failed."""
        videos = list(videos)
        return cls._build([(v.get("path", str(i)), v["img_names"]) for i, v in enumerate(videos)], videos, storage, device)

    @classmethod
    def from_videos(cls, videos, detector, batch_size: int = 32, storage: str = "device", device=None) -> "TrainDataCache":
        """preprocess.py and then the cache, on the device: videos yields one dict per video with "frames" ((F,H,W,3) uint8
        BGR, host memory or a CUDA tensor), "wav" (float samples, None = the audio failed), "sr" (default 16000) and "path".
        `detector` is this package's `face_detection.FaceAlignment`, `batch_size` preprocess.py's --batch_size.  Each video's
        kept frames are `face_crops`' crops, named "{i}.jpg" by frame index; its mel is melspectrogram(resample(wav, sr,
        16000)), as the Dataset's load_wav of the script's audio.wav gives it.  The frames are the 96x96 resize of the raw
        crop, without the reference's JPEG round trip (DESIGN.md section 3.12)."""
        import torch
        from . import audio
        dev = _cache_device(storage, device)

        def alloc(n):
            return torch.empty((n, IMG, IMG, 3), dtype=torch.uint8, device=dev) if storage == "device" else \
                torch.empty((n, IMG, IMG, 3), dtype=torch.uint8, pin_memory=True)
        buf, used, scan, decoded = alloc(0), 0, [], []
        for i, v in enumerate(videos):
            frames = v["frames"]
            F = len(frames)
            if used + F > buf.shape[0]:           # grow geometrically: the kernel writes straight into the cache
                nb = alloc(max(used + F, 2 * buf.shape[0]))
                nb[:used].copy_(buf[:used])
                buf = nb
            rows, _ = face_crops(detector, frames, batch_size, out=buf[used:used + F])
            names = ["{}.jpg".format(j) for j in np.flatnonzero(rows[:, 0] == 0)]
            wav, sr = v.get("wav"), int(v.get("sr", SAMPLE_RATE))
            if wav is not None and sr != SAMPLE_RATE:
                try:
                    w = wav if isinstance(wav, torch.Tensor) else torch.as_tensor(np.asarray(wav, dtype=np.float32))
                    wav = audio.resample(w.to(dev, torch.float32), sr, SAMPLE_RATE)
                except Exception:     # load_wav raises on such audio: the video keeps its frames and loses its audio
                    wav = None
            path = v.get("path", str(i))
            scan.append((path, names))
            decoded.append({"path": path, "img_names": names, "slots": range(used, used + len(names)), "wav": wav})
            used += len(names)
        if used != buf.shape[0]:
            buf = alloc(used).copy_(buf[:used])
        return cls._build(scan, decoded, storage, dev, frames=buf)

    @classmethod
    def _build(cls, scan, decoded, storage, device, frames=None):
        """frames: None (resize every decoded crop into a new cache), or the finished cache, whose slots each decoded
        video gives as "slots"."""
        import torch
        from . import _lib, audio
        dev = _cache_device(storage, device)
        n = sum(len(names) for _, names in scan)
        if n == 0:
            raise ValueError("the dataset has no *.jpg frames")
        shape = (n, IMG, IMG, 3)
        given = frames is not None
        if not given:
            frames = torch.zeros(shape, dtype=torch.uint8, device=dev) if storage == "device" else \
                torch.zeros(shape, dtype=torch.uint8).pin_memory()
        elif tuple(frames.shape) != shape:
            raise ValueError(f"expected a frame cache of shape {shape}, got {tuple(frames.shape)}")
        ctx = audio._context(dev.index)
        stream = torch.cuda.current_stream(dev)
        pending, canvas_hw = [], [0, 0]   # (slot, crop) waiting for the next resize launch, and their canvas's (h, w)

        def flush():
            if not pending:
                return
            hmax, wmax = canvas_hw
            canvas = np.zeros((len(pending), hmax, wmax, 3), dtype=np.uint8)
            boxes = np.zeros((len(pending), 5), dtype=np.int32)
            for k, (_, c) in enumerate(pending):
                canvas[k, :c.shape[0], :c.shape[1]] = c
                boxes[k] = (k, 0, c.shape[0], 0, c.shape[1])
            src = torch.from_numpy(canvas).to(dev)
            out = torch.empty((len(pending), IMG, IMG, 3), dtype=torch.uint8, device=dev)
            _lib.check(ctx.lib.w2l_crop_resize_u8(ctx.h, C.c_void_p(src.data_ptr()), len(pending), hmax, wmax,
                                                  boxes.ctypes.data_as(C.POINTER(C.c_int32)), len(pending),
                                                  C.c_void_p(out.data_ptr()), C.c_void_p(stream.cuda_stream)))
            idx = torch.tensor([s for s, _ in pending], dtype=torch.long)
            if storage == "device":
                frames[idx.to(dev)] = out
            else:
                frames[idx] = out.cpu()
            pending.clear()
            canvas_hw[:] = [0, 0]

        index, mels, slot, mel_off = [], [], 0, 0
        for (path, names), v in zip(scan, decoded):
            slots = [int(k) for k in v["slots"]] if given else []
            for c in ([] if given else v["crops"]):
                if c is None:
                    slots.append(-1)
                else:
                    c = np.asarray(c)
                    if c.dtype != np.uint8 or c.ndim != 3 or c.shape[2] != 3 or c.shape[0] == 0 or c.shape[1] == 0:
                        raise ValueError(f"{path}: expected uint8 (h, w, 3) BGR crops, got {c.dtype} {c.shape}")
                    h, w = max(canvas_hw[0], c.shape[0]), max(canvas_hw[1], c.shape[1])
                    if pending and (len(pending) + 1) * h * w * 3 > _CANVAS_BYTES:
                        flush()
                        h, w = c.shape[:2]
                    canvas_hw[:] = [h, w]
                    pending.append((slot + len(slots), c))
                    slots.append(slot + len(slots))
            if len(slots) != len(names):
                raise ValueError(f"{path}: {len(names)} names but {len(slots)} crops")
            mel = cls._orig_mel(v, dev)
            if mel is None:
                index.append(VideoIndex(path, names, slots, mel_off, -1))
            else:
                index.append(VideoIndex(path, names, slots, mel_off, mel.shape[0]))
                mels.append(mel)
                mel_off += mel.shape[0]
            slot += len(slots)
        flush()
        if mel_off + MEL_STEP > 2 ** 31 - 1:
            raise ValueError(f"{mel_off} mel rows: more than the int32 sample table addresses")
        mel_t = torch.cat(mels, 0).contiguous() if mels else torch.zeros((MEL_STEP, 80), device=dev)
        torch.cuda.current_stream(dev).synchronize()
        return cls(index, frames, mel_t, dev)

    @staticmethod
    def _orig_mel(v, dev):
        """`audio.melspectrogram(wav).T` as fp32 (rows, 80) on `dev`, or None where load_wav or the mel raised (the reference
        then rejects every draw of the video, wav2lip_train.py:136-142)."""
        import torch
        from . import audio
        if v.get("mel") is not None:
            m = torch.as_tensor(np.ascontiguousarray(v["mel"], dtype=np.float32)).to(dev)
            if m.dim() != 2 or m.shape[1] != 80:
                raise ValueError(f"expected an orig_mel of shape (rows, 80), got {tuple(m.shape)}")
            return m
        wav = v.get("wav")
        if wav is None:
            return None
        try:
            w = wav.to(dev, torch.float32) if isinstance(wav, torch.Tensor) and wav.is_cuda else \
                torch.as_tensor(np.asarray(wav, dtype=np.float32)).to(dev)
            return audio.melspectrogram(w).t().contiguous()
        except Exception:
            return None

    @property
    def n_frames(self) -> int:
        return int(self.frames.shape[0])

    @property
    def n_mel_rows(self) -> int:
        return int(self.mels.shape[0])


class _Batches:
    FIELDS = 0

    def __init__(self, cache: TrainDataCache, batch_size: int, rng=_random):
        if int(batch_size) <= 0:
            raise ValueError(f"batch_size must be positive, got {batch_size}")
        self.cache, self.batch_size, self.rng = cache, int(batch_size), rng

    def samples(self, n: int) -> np.ndarray:
        """The next n sample rows (int32), drawn as n `__getitem__` calls draw them."""
        return np.asarray([self._sample(self.cache.videos, self.rng) for _ in range(n)], dtype=np.int32).reshape(n, self.FIELDS)

    def next_batch(self, size: int = None):
        """One batch of `size` (default batch_size) samples: fresh CUDA tensors written on the current stream."""
        return self.assemble(self.samples(self.batch_size if size is None else int(size)))

    def epoch(self):
        """ceil(n_videos / B) batches, the last one short: len(Dataset) = len(all_videos), DataLoader drop_last=False."""
        n = len(self.cache.videos)
        for start in range(0, n, self.batch_size):
            yield self.next_batch(min(self.batch_size, n - start))

    def _call(self, fn, table, outs):
        import torch
        from . import _lib, audio
        table = np.ascontiguousarray(table, dtype=np.int32)
        if table.ndim != 2 or table.shape[1] != self.FIELDS or table.shape[0] == 0:
            raise ValueError(f"expected an (B, {self.FIELDS}) sample table, got {table.shape}")
        c = self.cache
        ctx = audio._context(c.device.index)
        stream = torch.cuda.current_stream(c.device).cuda_stream
        _lib.check(getattr(ctx.lib, fn)(ctx.h, C.c_void_p(c.frames.data_ptr()), c.n_frames, C.c_void_p(c.mels.data_ptr()),
                                        c.n_mel_rows, table.ctypes.data_as(C.POINTER(C.c_int32)), table.shape[0],
                                        *[C.c_void_p(o.data_ptr()) for o in outs], C.c_void_p(stream)))
        return outs


class Wav2LipBatches(_Batches):
    """wav2lip_train.py / hq_wav2lip_train.py batches: (x (B,6,5,96,96), indiv_mels (B,5,1,80,16), mel (B,1,80,16),
    gt (B,3,5,96,96)), fp32 CUDA tensors ready for `Wav2LipTrainStep` or the mirrors in train mode."""
    FIELDS = W2L_FIELDS
    _sample = staticmethod(sample_wav2lip)

    def assemble(self, table):
        import torch
        B, d = len(table), self.cache.device
        outs = (torch.empty((B, 6, SYNCNET_T, IMG, IMG), device=d), torch.empty((B, SYNCNET_T, 1, 80, MEL_STEP), device=d),
                torch.empty((B, 1, 80, MEL_STEP), device=d), torch.empty((B, 3, SYNCNET_T, IMG, IMG), device=d))
        return self._call("w2l_train_batch_wav2lip", table, outs)


class SyncNetBatches(_Batches):
    """color_syncnet_train.py batches: (x (B,15,48,96), mel (B,1,80,16), y (B,1)), fp32 CUDA tensors."""
    FIELDS = SYNC_FIELDS
    _sample = staticmethod(sample_syncnet)

    def assemble(self, table):
        import torch
        B, d = len(table), self.cache.device
        outs = (torch.empty((B, 3 * SYNCNET_T, IMG // 2, IMG), device=d), torch.empty((B, 1, 80, MEL_STEP), device=d),
                torch.empty((B, 1), device=d))
        return self._call("w2l_train_batch_syncnet", table, outs)
