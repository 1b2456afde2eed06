"""Generate tests/golden/preprocess.npz from the REAL reference preprocess.py:

    python tests/golden/make_golden_preprocess.py --reference PATH/TO/Wav2Lip

It imports the reference's preprocess.py by path (with sys.argv set, as its module-level argparse needs) and runs its
`mp_handler` -> `process_video_file` on scripted videos:
  * `cv2.VideoCapture` is replaced by a reader that yields the case's seeded frames;
  * `face_detection.FaceAlignment.__init__` is replaced BEFORE the module-level `fa = [...]` runs, so it only sets
    `self.face_detector` to a scripted object whose `detect_from_batch` returns the case's float32 (5,) rows.  The
    reference's own `get_detections_for_batch` still reverses the channels, clips and converts with int().  The reference's
    SFDDetector is never built (without s3fd.pth it would download the weights), `torch.utils.model_zoo.load_url` raises,
    and the import-time `s3fd.pth` check (relative to the current directory) finds an empty placeholder in a temporary cwd;
  * `cv2.imwrite` records each name and crop (shape, sha256 of the array and of the written jpg bytes) and then calls the
    real `imwrite` into a temporary directory, so empty crops raise for real;
  * `traceback.print_exc` inside the script records that mp_handler caught an exception (the video was abandoned).
The reference's audio.py imports librosa, which is not needed here: `sys.modules["audio"]` is an empty stand-in.

Stored (data only, no reference source), per case k:
  c{k}_frames (F,H,W,3) uint8   the video's BGR frames
  c{k}_has (F,) bool, c{k}_dets (F,5) float32   whether the scripted detector returned a box, and the box (x1 y1 x2 y2 s)
  c{k}_batch                    --batch_size
  c{k}_files                    the jpg names written, in order
  c{k}_shapes (n,3), c{k}_sha_arr, c{k}_sha_jpg   each written crop's shape, sha256 of its array bytes and of the jpg file
  c{k}_aborted                  whether mp_handler caught an exception
  case_names, cv2_version
"""
import argparse
import hashlib
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np

H, W = 64, 80
INF, NAN = np.float32(np.inf), np.float32(np.nan)


def frames_for(seed, F):
    """A wrapping gradient with sparse noise: every byte value and sharp edges, small once compressed."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    out = np.empty((F, H, W, 3), dtype=np.uint8)
    for f in range(F):
        base = (yy * 5 + xx * 3 + f * 7 + seed * 13)[..., None] + np.array([0, 85, 170])
        noise = rng.integers(0, 256, (H, W, 3)) * (rng.random((H, W, 1)) < 1 / 64)
        out[f] = (base + noise) % 256
    return out


def box(f):
    """The default box of frame f: inside the frame, a few pixels of drift."""
    return [4.5 + f % 5, 3.25 + (f * 3) % 7, 50.75 + f % 9, 58.5 - f % 4, 0.99]


def case(name, F, batch=32, none=(), boxes=None, seed=0):
    boxes = dict(boxes or {})
    has = np.array([f not in none for f in range(F)])
    dets = np.array([boxes.get(f, box(f)) if has[f] else [0, 0, 0, 0, 0] for f in range(F)], dtype=np.float32)
    return name, frames_for(seed, F), has, dets, batch


CASES = [
    case("no_face", 6, none=(1, 3), seed=1),
    case("negative", 5, boxes={2: [-5.5, -3.2, 40.7, 50.9, 0.9]}, seed=2),
    case("fractional", 5, boxes={0: [10.9, 7.99, 50.5, 60.01, 0.8], 3: [0.4, 0.6, 79.99, 63.999, 0.7]}, seed=3),
    case("past_frame", 5, boxes={1: [20.0, 30.0, 120.5, 99.0, 0.9], 4: [0.0, 0.0, 1e30, 1e30, 0.9]}, seed=4),
    case("start_past_right", 8, boxes={3: [85.0, 10.0, 100.0, 40.0, 0.9]}, seed=5),
    case("subpixel", 6, boxes={2: [10.2, 10.3, 10.8, 10.9, 0.9]}, seed=6),
    case("neg_inf", 4, boxes={1: [-INF, 5.0, 40.0, 50.0, 0.9], 2: [3.0, -INF, 40.0, 50.0, 0.9]}, seed=7),
    case("pos_inf", 70, none=(5, 40), boxes={37: [3.0, 4.0, INF, 50.0, 0.9]}, seed=8),
    case("nan", 40, boxes={5: [3.0, NAN, 40.0, 50.0, 0.9]}, seed=9),
    case("nan_score_only", 4, boxes={2: [3.0, 4.0, 40.0, 50.0, NAN]}, seed=10),
    case("empty_then_nan_same_batch", 40, boxes={33: [3.0, 4.0, 3.0, 50.0, 0.9], 36: [NAN, 4.0, 40.0, 50.0, 0.9]}, seed=11),
    case("empty_then_nan_later_batch", 40, boxes={10: [3.0, 70.0, 40.0, 90.0, 0.9], 36: [NAN, 4.0, 40.0, 50.0, 0.9]}, seed=12),
    case("nan_then_empty_same_batch", 40, boxes={33: [NAN, 4.0, 40.0, 50.0, 0.9], 36: [3.0, 4.0, 3.0, 50.0, 0.9]}, seed=13),
    case("len1", 1, seed=14),
    case("len31", 31, none=(0, 30), seed=15),
    case("len32", 32, none=(31,), seed=16),
    case("len33", 33, none=(32,), seed=17),
    case("len70", 70, none=(3, 33, 64), seed=18),
    case("batch4", 18, batch=4, none=(2,), boxes={9: [3.0, 4.0, INF, 50.0, 0.9]}, seed=19),
]


class _Capture:
    def __init__(self, frames):
        self.frames, self.i = frames, 0

    def read(self):
        if self.i >= len(self.frames):
            return False, None
        self.i += 1
        return True, self.frames[self.i - 1].copy()

    def release(self):
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "preprocess.npz"))
    a = ap.parse_args()
    ref = os.path.abspath(a.reference)
    import cv2
    import torch.utils.model_zoo

    def no_download(*args, **kw):
        raise RuntimeError("make_golden_preprocess must not download anything")
    torch.utils.model_zoo.load_url = no_download

    current = {}

    class Scripted:
        def detect_from_batch(self, images):
            start = current["at"]
            current["at"] += len(images)
            return [[current["dets"][f].copy()] if current["has"][f] else [] for f in range(start, start + len(images))]

    sys.path.insert(0, ref)
    sys.modules["audio"] = types.ModuleType("audio")
    import face_detection
    assert os.path.dirname(face_detection.__file__).startswith(ref), face_detection.__file__

    def fa_init(self, *args, **kw):
        self.face_detector = Scripted()
    face_detection.FaceAlignment.__init__ = fa_init

    real_imwrite, real_capture = cv2.imwrite, cv2.VideoCapture
    written = []

    def imwrite(path, img):
        ok = real_imwrite(path, img)
        with open(path, "rb") as f:
            jpg = f.read()
        written.append((os.path.basename(path), img.shape, hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest(),
                        hashlib.sha256(jpg).hexdigest()))
        return ok

    out = {"case_names": np.array([c[0] for c in CASES]), "cv2_version": np.array(cv2.__version__)}
    with tempfile.TemporaryDirectory() as cwd, tempfile.TemporaryDirectory() as dst:
        os.makedirs(os.path.join(cwd, "face_detection", "detection", "sfd"))
        open(os.path.join(cwd, "face_detection", "detection", "sfd", "s3fd.pth"), "wb").close()
        old = os.getcwd()
        os.chdir(cwd)
        try:
            cv2.imwrite = imwrite
            for k, (name, frames, has, dets, batch) in enumerate(CASES):
                sys.argv = ["preprocess.py", "--data_root", "unused", "--preprocessed_root", dst, "--batch_size", str(batch)]
                spec = importlib.util.spec_from_file_location(f"ref_preprocess_{k}", os.path.join(ref, "preprocess.py"))
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                caught = []
                mod.traceback = types.SimpleNamespace(print_exc=lambda: caught.append(sys.exc_info()[1]))
                cv2.VideoCapture = lambda path, frames=frames: _Capture(frames)
                current.update(at=0, dets=dets, has=has)
                written.clear()
                mod.mp_handler((f"videos/set/{name}.mp4", mod.args, 0))
                out[f"c{k}_frames"], out[f"c{k}_has"], out[f"c{k}_dets"] = frames, has, dets
                out[f"c{k}_batch"] = np.int32(batch)
                out[f"c{k}_files"] = np.array([w[0] for w in written], dtype="<U16")
                out[f"c{k}_shapes"] = np.array([w[1] for w in written], dtype=np.int32).reshape(-1, 3)
                out[f"c{k}_sha_arr"] = np.array([w[2] for w in written], dtype="<U64")
                out[f"c{k}_sha_jpg"] = np.array([w[3] for w in written], dtype="<U64")
                out[f"c{k}_aborted"] = np.bool_(bool(caught))
                print(f"{name}: {len(written)} files, aborted={bool(caught)} {caught[0]!r}" if caught else
                      f"{name}: {len(written)} files")
        finally:
            cv2.imwrite, cv2.VideoCapture = real_imwrite, real_capture
            os.chdir(old)
    np.savez_compressed(a.out, **out)
    print("wrote", a.out, os.path.getsize(a.out), "bytes")


if __name__ == "__main__":
    main()
