"""Golden vectors for the resize rows (SURVEY.md section 8 f2) from OpenCV ITSELF (cv2 is importable in the build
container; opencv-python is the reference's own dependency, requirements.txt): `cv2.resize(img, dsize)` with the default
INTER_LINEAR on seeded uint8 images, for the two call shapes of inference.py (:126 crop -> 96x96, :269 96x96 -> box) plus
odd cases (1-pixel sources, exact 2x, extreme aspect).

resize.npz holds the outputs of small cases.  resize_video.json holds, for crops and pastes at video frame sizes (720p,
1080p, 4K and an odd 1079x1917), the SHA-256 of cv2's output bytes: the seeded frames are regenerated where the digests
are checked, so megabytes of random bytes stay out of git.  Run:
    python tests/golden/make_golden_resize.py          # both files
    python tests/golden/make_golden_resize.py video    # resize_video.json only"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = [  # (src_h, src_w, dst_h, dst_w)
    (137, 121, 96, 96), (96, 96, 137, 121), (192, 192, 96, 96), (48, 48, 96, 96), (96, 96, 96, 96), (1, 1, 96, 96),
    (96, 96, 1, 1), (5, 300, 96, 96), (96, 96, 301, 7), (250, 211, 96, 96), (96, 96, 211, 250), (33, 97, 96, 96),
]

# crop: cv2.resize(image(H, W, seed)[y1:y2, x1:x2], (96, 96)); paste: cv2.resize(image(96, 96, seed), (w, h))
VIDEO_CROPS = [  # ((H, W), seed, (y1, y2, x1, x2))
    ((720, 1280), 2000, (210, 510, 500, 760)),       # a face
    ((720, 1280), 2001, (0, 720, 0, 1280)),          # the whole frame
    ((720, 1280), 2002, (540, 720, 1100, 1280)),     # bottom-right corner
    ((1080, 1920), 2003, (200, 800, 700, 1240)),     # a large face
    ((1080, 1920), 2004, (0, 150, 0, 150)),          # top-left corner
    ((1080, 1920), 2005, (500, 508, 300, 1200)),     # an 8 x 900 sliver
    ((1080, 1920), 2006, (700, 701, 100, 400)),      # 1 px tall
    ((1080, 1920), 2007, (100, 400, 1919, 1920)),    # 1 px wide, on the right edge
    ((2160, 3840), 2008, (1000, 1900, 2900, 3800)),  # a 900 px face
    ((2160, 3840), 2009, (0, 2160, 0, 3840)),        # the whole 4K frame
    ((2160, 3840), 2010, (2100, 2160, 3760, 3840)),  # 60 x 80: upscaled to 96, bottom-right corner
    ((1079, 1917), 2011, (379, 1079, 1267, 1917)),   # odd frame, bottom-right corner
    ((1079, 1917), 2012, (40, 137, 800, 895)),       # 97 x 95
]
VIDEO_PASTES = [  # (seed, (h, w))
    (2100, (900, 900)), (2101, (1079, 1917)), (2102, (2160, 3840)), (2103, (8, 900)), (2104, (900, 8)),
    (2105, (1, 300)), (2106, (300, 1)), (2107, (150, 170)), (2108, (95, 97)), (2109, (97, 95)),
]


def image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


def write_npz():
    out = {"cases": np.array(CASES, dtype=np.int32), "cv2_version": np.array(cv2.__version__)}
    for i, (sh, sw, dh, dw) in enumerate(CASES):
        out[f"out{i}"] = cv2.resize(image(sh, sw, 1000 + i), (dw, dh))
    # the paste: one frame, two boxes
    frames = np.random.default_rng(7).integers(0, 256, (2, 120, 160, 3), dtype=np.uint8)
    boxes = np.array([[0, 10, 100, 20, 95], [1, 0, 120, 33, 160], [1, 57, 58, 3, 4]], dtype=np.int32)
    pred = np.random.default_rng(8).integers(0, 256, (3, 96, 96, 3), dtype=np.uint8)
    crops, pasted = [], []
    for p, (f, y1, y2, x1, x2) in zip(pred, boxes):
        crops.append(cv2.resize(frames[f][y1:y2, x1:x2], (96, 96)))
        fr = frames[f].copy()
        fr[y1:y2, x1:x2] = cv2.resize(p, (x2 - x1, y2 - y1))
        pasted.append(fr)
    out["boxes"] = boxes
    out["crops"] = np.stack(crops)
    out["pasted"] = np.stack(pasted)
    np.savez_compressed(os.path.join(HERE, "resize.npz"), **out)
    print("wrote resize.npz", {k: getattr(v, "shape", None) for k, v in out.items()})


def write_video_json():
    cases = []
    for (H, W), seed, (y1, y2, x1, x2) in VIDEO_CROPS:
        out = cv2.resize(image(H, W, seed)[y1:y2, x1:x2], (96, 96))
        cases.append({"kind": "crop", "frame": [H, W], "seed": seed, "box": [y1, y2, x1, x2], "sha256": digest(out)})
    for seed, (h, w) in VIDEO_PASTES:
        out = cv2.resize(image(96, 96, seed), (w, h))
        assert out.shape == (h, w, 3)
        cases.append({"kind": "paste", "seed": seed, "size": [h, w], "sha256": digest(out)})
    with open(os.path.join(HERE, "resize_video.json"), "w") as f:   # one case per line
        f.write('{"cv2_version": %s, "cases": [\n' % json.dumps(cv2.__version__))
        f.write(",\n".join(json.dumps(c) for c in cases))
        f.write("\n]}\n")
    print("wrote resize_video.json:", len(cases), "cases")


if __name__ == "__main__":
    what = sys.argv[1:] or ["npz", "video"]
    if "npz" in what:
        write_npz()
    if "video" in what:
        write_video_json()
