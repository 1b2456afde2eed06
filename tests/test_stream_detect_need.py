"""Which frames a detecting session must have detected (include/w2l.h w2l_stream_detect_need, host code, no GPU): for
random videos, frame rates, smoothing and push splits, with audio shorter than, as long as and longer than the video,
`need` after each push never decreases, stays within F, is 1 for a still image and equals n_total at the end; the rows
the audio fixes (w2l_stream_schedule) do not change when the rects of frames at or past `need` are replaced, and do
change when frame need - 1 moves by 5 pixels, so the prefix is the smallest that holds every rect those rows read."""
import numpy as np
import pytest

from oracle.pipeline_oracle import mel_chunks
from wav2lip_b200 import stream

H, W = 72, 88
FPS = (25.0, 30.0, 29.97002997)


def _rects(rng, F):
    """Boxes well inside the frame, so that a 5-pixel move is not absorbed by the padding's clip."""
    x1, y1 = rng.integers(10, 40, F), rng.integers(10, 30, F)
    return np.stack([x1, y1, x1 + rng.integers(8, 20, F), y1 + rng.integers(8, 20, F)], 1).astype(np.int64)


def _splits(rng, n):
    out, left = [], n
    while left:
        k = int(min(left, rng.integers(1, 4000)))
        out.append(k)
        left -= k
    return out


def _rows(L, F, fps, rects, nosmooth, final):
    return stream.schedule(L, F, H, W, fps, rects=rects, nosmooth=nosmooth, final=final)[1]


def _check_minimal(L, F, fps, rects, nosmooth, final, need, rng):
    rows = _rows(L, F, fps, rects, nosmooth, final)
    other = rects.copy()
    other[need:] = _rects(rng, F)[need:]
    assert np.array_equal(_rows(L, F, fps, other, nosmooth, final), rows), (L, need)
    if len(rows) == 0:
        return
    moved = rects.copy()
    moved[need - 1] += 5
    assert not np.array_equal(_rows(L, F, fps, moved, nosmooth, final), rows), (L, need)


@pytest.mark.parametrize("seed", range(24))
def test_need_is_a_minimal_monotone_prefix(seed):
    rng = np.random.default_rng(seed)
    F = int(rng.choice([1, 2, 3, 4, 5, 6, 9, 17, 40]))
    fps = float(FPS[seed % 3])
    nosmooth = bool(seed % 2)
    ratio = (0.5, 1.0, 2.0)[(seed // 2) % 3]                 # audio shorter than, as long as, longer than the video
    L_end = max(3300, int(ratio * F / fps * 16000) + int(rng.integers(0, 300)))
    rects = _rects(rng, F)
    last, L = 0, 0
    for piece in _splits(rng, L_end):
        L += piece
        need = stream.detect_need(L, F, H, W, fps, nosmooth=nosmooth)
        assert last <= need <= F, (L, last, need)
        if F == 1:
            assert need == 1
        if need:
            _check_minimal(L, F, fps, rects, nosmooth, False, need, rng)
        last = need
    need = stream.detect_need(L_end, F, H, W, fps, nosmooth=nosmooth, final=True)
    n_total = min(len(mel_chunks(np.zeros((80, 1 + L_end // 200)), fps)), F)
    assert last <= need == n_total, (last, need, n_total)
    _check_minimal(L_end, F, fps, rects, nosmooth, True, need, rng)


def test_need_of_the_open_and_ahead_windows():
    """The constants of the server's prefetch at 25 fps: 400 ms of audio fix 2 smoothed rows (frames 0-5)."""
    assert stream.detect_need(6400, 250, H, W, 25.0) == 6
    assert stream.detect_need(6400, 250, H, W, 25.0, nosmooth=True) == 5
    assert stream.detect_need(0, 250, H, W, 25.0) == 0
    assert stream.detect_need(0, 1, H, W, 25.0) == 1


def test_need_rejects_a_fixed_box():
    from wav2lip_b200 import _lib
    d = stream._desc(10, H, W, 25.0, (0, 10, 0, 0), False, (5, 60, 7, 80))
    import ctypes as C
    n = C.c_int64()
    assert _lib.get_lib().w2l_stream_detect_need(C.byref(d), 16000, 0, C.byref(n)) == _lib.W2L_EINVAL
