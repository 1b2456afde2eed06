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
    def _build(cls, scan, decoded, storage, device):
        import torch
        from . import _lib, audio
        if storage not in ("device", "pinned"):
            raise ValueError(f"storage must be 'device' or 'pinned', got {storage!r}")
        dev = torch.device("cuda", torch.cuda.current_device() if device is None else torch.device(device).index or 0)
        n = sum(len(names) for _, names in scan)
        if n == 0:
            raise ValueError("the dataset has no *.jpg frames")
        shape = (n, IMG, IMG, 3)
        frames = torch.zeros(shape, dtype=torch.uint8, device=dev) if storage == "device" else \
            torch.zeros(shape, dtype=torch.uint8).pin_memory()
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
            slots = []
            for c in v["crops"]:
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
            return audio.melspectrogram(torch.as_tensor(np.asarray(wav, dtype=np.float32)).to(dev)).t().contiguous()
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
