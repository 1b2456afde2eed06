"""NumPy restatement of the reference training Datasets' tensor construction, for tests/test_train_data.py and
tests/test_gpu_train_data.py (not a test module itself).

Given the sampled rows of wav2lip_b200.data (frame slots, absolute mel rows, label) and the cache's contents, this builds what
`default_collate` of the `__getitem__` calls returns, with the reference's statements as they are written:
  wav2lip_train.py:101-106 prepare_window, :152-163 (mask rows H//2.., concat, torch.FloatTensor), :75-99 the mel windows;
  color_syncnet_train.py:121-131 (concat along channels, / 255., transpose, lower half).
It also rebuilds the cache's index from the golden fixture (tests/golden/train_data.npz).
"""
import hashlib

import numpy as np

from oracle.pipeline_oracle import resize_linear_u8


def fixture_videos(g, mels=True):
    """The fixture as `TrainDataCache.from_arrays` input: names in glob order, imread arrays (None: unreadable), orig_mel."""
    shapes, flat = g["crop_shapes"], g["crops_flat"]
    out, k, pos, moff = [], 0, 0, 0
    mel_flat = g["mel_flat"]
    for i, _ in enumerate(g["video_names"]):
        names = [str(n) for n in g[f"v{i}_names"]]
        crops = []
        for _ in names:
            h, w, c = (int(v) for v in shapes[k])
            k += 1
            if h < 0:
                crops.append(None)
            else:
                crops.append(flat[pos:pos + h * w * c].reshape(h, w, c))
                pos += h * w * c
        n_mel = int(g["mel_lens"][i])
        v = {"img_names": names, "crops": crops}
        if n_mel >= 0:
            v["mel"] = mel_flat[moff:moff + n_mel]
            moff += n_mel
        out.append(v)
    return out


def fixture_index(videos):
    """The cache's host index (wav2lip_b200.data.VideoIndex) of `fixture_videos`: one slot per name in order, -1 unreadable."""
    from wav2lip_b200.data import VideoIndex
    index, slot, moff = [], 0, 0
    for i, v in enumerate(videos):
        slots = [slot + j if c is not None else -1 for j, c in enumerate(v["crops"])]
        n_mel = len(v["mel"]) if "mel" in v else -1
        index.append(VideoIndex(str(i), v["img_names"], slots, moff, n_mel))
        slot += len(v["crops"])
        moff += max(n_mel, 0)
    return index


def cache_arrays(videos):
    """(frames (n,96,96,3) uint8 = cv2.resize(crop, (96, 96)) restated, zeros where unreadable; mels (rows, 80) fp32)."""
    frames = [resize_linear_u8(c, (96, 96)) if c is not None else np.zeros((96, 96, 3), np.uint8)
              for v in videos for c in v["crops"]]
    mels = [np.asarray(v["mel"], np.float32) for v in videos if "mel" in v]
    return np.stack(frames), np.concatenate(mels)


def wav2lip_batch(frames, mels, rows):
    """wav2lip_train.py:143-163 for each row, stacked: (x, indiv_mels, mel, gt)."""
    xs, ims, ms, ys = [], [], [], []
    for r in rows:
        def prepare_window(slots):
            x = np.asarray([frames[s] for s in slots]) / 255.
            return np.transpose(x, (3, 0, 1, 2))
        window = prepare_window(r[0:5])
        y = window.copy()
        window[:, :, window.shape[2] // 2:] = 0.
        wrong_window = prepare_window(r[5:10])
        x = np.concatenate([window, wrong_window], axis=0)
        mel = mels[r[10]:r[10] + 16]
        indiv = np.asarray([mels[s:s + 16].T for s in r[11:16]])
        xs.append(np.float32(x)); ims.append(np.float32(indiv)[:, None]); ms.append(np.float32(mel.T)[None]); ys.append(np.float32(y))
    return np.stack(xs), np.stack(ims), np.stack(ms), np.stack(ys)


def syncnet_batch(frames, mels, rows):
    """color_syncnet_train.py:121-131 for each row, stacked: (x, mel, y)."""
    xs, ms, ys = [], [], []
    for r in rows:
        window = [frames[s] for s in r[0:5]]
        x = np.concatenate(window, axis=2) / 255.
        x = x.transpose(2, 0, 1)
        x = x[:, x.shape[1] // 2:]
        mel = mels[r[5]:r[5] + 16]
        xs.append(np.float32(x)); ms.append(np.float32(mel.T)[None]); ys.append(np.ones(1, np.float32) * r[6])
    return np.stack(xs), np.stack(ms), np.stack(ys)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


class LogRandom:
    """A random.Random whose randint / choice calls are logged as the fixture logs them: (0 randint | 1 choice, n, index)."""

    def __init__(self, seed):
        import random
        self.r, self.log = random.Random(seed), []

    def randint(self, a, b):
        v = self.r.randint(a, b)
        self.log.append((0, b + 1, v))
        return v

    def choice(self, seq):
        v = self.r.choice(seq)
        self.log.append((1, len(seq), list(seq).index(v)))
        return v
