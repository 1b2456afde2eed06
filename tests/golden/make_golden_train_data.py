"""Generate tests/golden/train_data.npz from the REAL reference training datasets:

    python tests/golden/make_golden_train_data.py --reference PATH/TO/Wav2Lip

It writes a small preprocessed dataset to a temporary directory (frame crops named `<id>.jpg` and `audio.wav` per video) with a
`filelists/train.txt` in a temporary current directory, imports the reference's wav2lip_train.py and color_syncnet_train.py by
path (with sys.argv set, as their module-level argparse needs), and calls `Dataset("train").__getitem__` through a
`DataLoader(batch_size=B, num_workers=0)` for several seeds, with the scripts' `random` module replaced by a logging proxy.

The reference's audio.py imports librosa, which is not installed where this runs, so `sys.modules["audio"]` is a shim: a
scipy.io.wavfile `load_wav` (16-bit PCM / 32768, the files are written at 16 kHz so nothing is resampled) and
`oracle.mel_oracle.melspectrogram` (the repository's NumPy restatement of audio.melspectrogram).  The mels it produced are stored,
so the fixture pins the mel windows given that `orig_mel`.

The frames are PNG-encoded under `.jpg` names: cv2.imread decodes by content, so the decoded arrays are exact and a test can
rebuild the directory byte for byte.  Stored (data only, no reference source):
  video_names, v{i}_names         each video's directory name and its jpg names in the order glob returned them
  crops_flat, crop_shapes         every name's cv2.imread array (shape -1: unreadable), videos in filelist order
  mel_flat, mel_lens              each video's orig_mel = melspectrogram(wav).T (mel_lens -1: the audio failed)
  {ds}_s{seed}_log                the draw log: rows (0 randint | 1 choice, n, result index)
  {ds}_s{seed}_picks              per sample: (video, img_name index, wrong_img_name index, label (syncnet) or -1)
  {ds}_s{seed}_b{B}_sha           per batch, sha256 of each output tensor's float32 bytes (wav2lip: x, indiv_mels, mel, gt;
                                  syncnet: x, mel, y)
Dataset content covers: a video with <= 15 frames, a missing frame id, a zero-byte jpg, a video without audio.wav, a wav short
enough that late windows fail the 16-row rule, frame id 0, crops smaller than, larger than and not the shape of 96x96.
"""
import argparse
import hashlib
import importlib.util
import os
import random
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import mel_oracle as M  # noqa: E402

SEEDS = (0, 1, 7)
BATCHES = (1, 4, 16)

# (frames, crop h, crop w, wav seconds or None, missing ids, zero-byte ids)
VIDEOS = [
    (20, 40, 48, 1.1, (), ()),
    (12, 40, 40, 1.0, (), ()),          # <= 15 frames: always redrawn
    (20, 36, 52, 1.1, (7,), ()),        # id 7 missing
    (20, 44, 38, 1.0, (), (10,)),       # 10.jpg is zero bytes
    (17, 40, 48, None, (), ()),         # no audio.wav
    (24, 48, 40, 0.6, (), ()),          # 49 mel rows: windows past frame 10 are short
    (16, 100, 98, 1.0, (), ()),         # larger than 96x96
    (16, 96, 96, 1.0, (), ()),          # exactly 96x96
    (17, 20, 30, 1.0, (), ()),          # small, wide
    (17, 64, 24, 1.0, (), ()),          # tall
]


class LogRandom:
    """The `random` calls the Dataset makes, logged."""

    def __init__(self, seed):
        self.r, self.log = random.Random(seed), []

    def randint(self, a, b):
        v = self.r.randint(a, b)
        self.log.append((0, b + 1, v))
        return v

    def choice(self, seq):
        v = self.r.choice(seq)
        self.log.append((1, len(seq), list(seq).index(v)))
        return v


def audio_shim():
    from scipy.io import wavfile
    mod = types.ModuleType("audio")

    def load_wav(path, sr):
        rate, data = wavfile.read(path)
        assert rate == sr
        return data.astype(np.float32) / np.float32(32768)

    mod.load_wav = load_wav
    mod.melspectrogram = M.melspectrogram
    return mod


def make_dataset(data_root, cwd):
    import cv2
    from scipy.io import wavfile
    rng = np.random.default_rng(2024)
    names = []
    for i, (n, h, w, secs, missing, zero) in enumerate(VIDEOS):
        vid = f"vid{i:02d}"
        d = os.path.join(data_root, vid)
        os.makedirs(d)
        names.append(vid)
        for fid in range(n):
            if fid in missing:
                continue
            p = os.path.join(d, f"{fid}.jpg")
            if fid in zero:
                open(p, "wb").close()
                continue
            # a wrapping gradient (every byte value, sharp edges) with noise on one pixel in 32: varied enough for the
            # resize and the /255, and compressible enough to keep the fixture small
            yy, xx = np.mgrid[0:h, 0:w]
            base = (yy * 7 + xx * 3 + fid * 11 + i * 29)[..., None] + np.array([0, 85, 170])
            noise = rng.integers(0, 256, (h, w, 3)) * (rng.random((h, w, 1)) < 1 / 32)
            img = ((base + noise) % 256).astype(np.uint8)
            ok, buf = cv2.imencode(".png", img)
            assert ok
            with open(p, "wb") as f:
                f.write(buf.tobytes())
        if secs is not None:
            wav = M.make_wav(int(secs * 16000), seed=100 + i, kind="mix")
            wavfile.write(os.path.join(d, "audio.wav"), 16000, (np.clip(wav, -1, 1) * 32767).astype(np.int16))
    os.makedirs(os.path.join(cwd, "filelists"))
    with open(os.path.join(cwd, "filelists", "train.txt"), "w") as f:
        for v in names:
            f.write(v + (" extra\n" if v.endswith("3") else "\n"))   # get_image_list keeps the first word
    return names


def load_script(ref, fname, data_root, ckpt):
    sys.argv = [fname, "--data_root", data_root, "--checkpoint_dir", ckpt]
    if fname == "wav2lip_train.py":
        sys.argv += ["--syncnet_checkpoint_path", "unused"]
    spec = importlib.util.spec_from_file_location("ref_" + fname[:-3], os.path.join(ref, fname))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.numpy(), dtype=np.float32).tobytes()).hexdigest()


def picks_of(log, syncnet):
    """The accepted draw of one sample: (video, img_name index, wrong_img_name index, label or -1)."""
    k = max(i for i, r in enumerate(log) if r[0] == 0)
    c = [r[2] for r in log[k + 1:]]
    if syncnet:
        return [log[k][2], c[0], c[-2], 1 - c[-1]]       # choice([True, False]) index 0 is y = 1
    return [log[k][2], c[0], c[-1], -1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="a checkout of the reference Wav2Lip repository")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "train_data.npz"))
    args = ap.parse_args()
    ref = os.path.abspath(args.reference)
    sys.path.insert(0, ref)
    sys.modules["audio"] = audio_shim()
    from torch.utils.data import DataLoader
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        data_root, cwd = os.path.join(tmp, "data"), os.path.join(tmp, "cwd")
        os.makedirs(data_root)
        os.makedirs(cwd)
        vids = make_dataset(data_root, cwd)
        prev = os.getcwd()
        os.chdir(cwd)
        try:
            w2l = load_script(ref, "wav2lip_train.py", data_root, tmp)
            sync = load_script(ref, "color_syncnet_train.py", data_root, tmp)
            import cv2
            from glob import glob
            ds_w, ds_s = w2l.Dataset("train"), sync.Dataset("train")
            assert ds_w.all_videos == [os.path.join(data_root, v) for v in vids]
            crops, shapes, mels, mel_lens = [], [], [], []
            out["video_names"] = np.array(vids)
            for i, vdir in enumerate(ds_w.all_videos):
                names = [os.path.basename(p) for p in glob(os.path.join(vdir, "*.jpg"))]
                out[f"v{i}_names"] = np.array(names)
                for n in names:
                    img = cv2.imread(os.path.join(vdir, n))
                    shapes.append(img.shape if img is not None else (-1, -1, -1))
                    if img is not None:
                        crops.append(img.reshape(-1))
                try:
                    m = sys.modules["audio"].melspectrogram(sys.modules["audio"].load_wav(os.path.join(vdir, "audio.wav"), 16000)).T
                    mels.append(np.asarray(m, dtype=np.float32))
                    mel_lens.append(m.shape[0])
                except Exception:
                    mel_lens.append(-1)
            out["crops_flat"] = np.concatenate(crops)
            out["crop_shapes"] = np.array(shapes, dtype=np.int32)
            out["mel_flat"] = np.concatenate(mels)
            out["mel_lens"] = np.array(mel_lens, dtype=np.int32)
            for tag, mod, ds in (("w2l", w2l, ds_w), ("sync", sync, ds_s)):
                for s in SEEDS:
                    for B in BATCHES:
                        proxy = LogRandom(s)
                        mod.random = proxy
                        shas, picks, mark = [], [], 0
                        for batch in DataLoader(ds, batch_size=B, num_workers=0):
                            shas.append([sha(t) for t in batch])
                        if B == 1:
                            # one sample per batch: split the log at each returned sample
                            proxy2 = LogRandom(s)
                            mod.random = proxy2
                            for _ in range(len(ds)):
                                ds[0]
                                p = picks_of(proxy2.log[mark:], tag == "sync")
                                mark = len(proxy2.log)
                                picks.append(p)
                            assert proxy2.log == proxy.log
                            out[f"{tag}_s{s}_log"] = np.array(proxy.log, dtype=np.int64)
                            out[f"{tag}_s{s}_picks"] = np.array(picks, dtype=np.int64)
                        out[f"{tag}_s{s}_b{B}_sha"] = np.array(shas)
                        print(tag, s, B, len(shas), "batches", len(proxy.log), "draws")
        finally:
            os.chdir(prev)
    np.savez_compressed(args.out, **out)
    print(args.out, os.path.getsize(args.out), "bytes")


if __name__ == "__main__":
    main()
