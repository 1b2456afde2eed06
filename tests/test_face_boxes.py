"""`wav2lip_b200.face_detection.face_boxes` (CPU): the padding, clipping and temporal smoothing of inference.py:87-103
on the detector's rectangles, against the reference's lines restated verbatim below (plain NumPy: get_smoothened_boxes
:60-67 and face_detect :87-103 without the detector call, the image crops and the debug image write)."""
import numpy as np
import pytest

from wav2lip_b200.face_detection import face_boxes


def _get_smoothened_boxes(boxes, T):                      # inference.py:60-67
    for i in range(len(boxes)):
        if i + T > len(boxes):
            window = boxes[len(boxes) - T:]
        else:
            window = boxes[i: i + T]
        boxes[i] = np.mean(window, axis=0)
    return boxes


def _reference(predictions, H, W, pads, nosmooth):      # inference.py:87-103
    results = []
    pady1, pady2, padx1, padx2 = pads
    for rect in predictions:
        if rect is None:
            raise ValueError('Face not detected! Ensure the video contains a face in all the frames.')

        y1 = max(0, rect[1] - pady1)
        y2 = min(H, rect[3] + pady2)
        x1 = max(0, rect[0] - padx1)
        x2 = min(W, rect[2] + padx2)

        results.append([x1, y1, x2, y2])

    boxes = np.array(results)
    if not nosmooth: boxes = _get_smoothened_boxes(boxes, T=5)  # noqa: E701
    return [(y1, y2, x1, x2) for (x1, y1, x2, y2) in boxes]


def _rects(rng, F, H, W):
    out = []
    for _ in range(F):
        x1, y1 = int(rng.integers(0, W - 8)), int(rng.integers(0, H - 8))
        out.append((x1, y1, int(rng.integers(x1 + 1, W + 20)), int(rng.integers(y1 + 1, H + 20))))
    return out


@pytest.mark.parametrize("F", [1, 2, 3, 4, 5, 6, 9, 40])
@pytest.mark.parametrize("nosmooth", [False, True])
@pytest.mark.parametrize("pads", [(0, 10, 0, 0), (7, 0, 13, 5), (40, 40, 40, 40)])
def test_face_boxes_matches_inference_py(F, nosmooth, pads):
    rng = np.random.default_rng(F * 31 + sum(pads) + nosmooth)
    H, W = 180, 320
    rects = _rects(rng, F, H, W)
    got = face_boxes(rects, H, W, pads=pads, nosmooth=nosmooth)
    ref = np.array(_reference(rects, H, W, pads, nosmooth))
    assert got.shape == (F, 4) and got.dtype.kind == "i"
    assert np.array_equal(got, ref)


def test_smoothing_quirks():
    # truncation of the mean into the integer array, and a tail window that includes already smoothed rows
    rects = [(0, 0, 10, 10), (1, 0, 11, 10), (0, 0, 10, 10), (0, 0, 10, 10), (0, 0, 10, 10), (5, 0, 15, 10), (9, 0, 19, 10)]
    got = face_boxes(rects, 100, 100, pads=(0, 0, 0, 0))
    assert got[0, 2] == 0                     # mean x1 of rows 0..4 = 0.2 -> 0
    assert np.array_equal(got, np.array(_reference(rects, 100, 100, (0, 0, 0, 0), False)))
    # fewer frames than the window: boxes[len - 5:] starts at a negative index
    rects = [(0, 0, 10, 10), (20, 0, 30, 10), (40, 0, 50, 10)]
    got = face_boxes(rects, 100, 100, pads=(0, 0, 0, 0))
    assert np.array_equal(got, np.array(_reference(rects, 100, 100, (0, 0, 0, 0), False)))


def test_missing_face_names_the_frame():
    rects = [(0, 0, 10, 10), None, (0, 0, 10, 10)]
    with pytest.raises(ValueError, match="frame 1"):
        face_boxes(rects, 100, 100)
    with pytest.raises(ValueError):
        _reference(rects, 100, 100, (0, 10, 0, 0), False)
