"""The streaming session's schedule (include/w2l.h w2l_stream_schedule, host code, no GPU): for random utterances and
random push splits the rows each push fixes form a gap-free prefix, obey the finality rules of DESIGN.md section 3.8,
and concatenated equal the offline rows of inference.py (tests/stream_offline.py).  Also pins rule 1 (when a mel frame
is final) against the reference's own arithmetic (oracle/mel_oracle.py) on prefixes of a wav."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from stream_offline import offline_rows, random_rects  # noqa: E402
from wav2lip_b200 import stream  # noqa: E402

H, W = 72, 88
FPS = (25.0, 30.0, 29.97002997)


def _mel_final(L):
    return (L - 400) // 200 + 1 if L >= 400 else 0


def _expected_fixed(L, fps, F, fixed_box):
    """Rules 1-3 restated independently of the C code: the count of rows L samples fix."""
    M = _mel_final(L)
    n_reg = 0
    while int(n_reg * (80. / fps)) + 16 <= M:
        n_reg += 1
    n_lb = n_reg + 1 if n_reg else 0
    if fixed_box or n_lb >= F:
        return n_reg
    return max(0, min(n_reg, n_lb - 4))


def _splits(rng, L_end, kind):
    if kind == "one":
        return [L_end]
    if kind == "ones":
        return [1] * L_end
    if kind == "640":
        return [640] * (L_end // 640) + ([L_end % 640] if L_end % 640 else [])
    out, left = [], L_end
    while left:
        k = int(min(left, rng.integers(1, 4000)))
        out.append(k)
        left -= k
    return out


def _run(L_end, fps, F, nosmooth, box, kind, seed):
    rng = np.random.default_rng(seed)
    rects = random_rects(rng, F, H, W)
    kw = dict(rects=None if box else rects, nosmooth=nosmooth, box=box)
    try:
        ref = offline_rows(L_end, fps, F, H, W, **kw)
    except ValueError:
        ref = None
    got, L = [], 0
    for piece in _splits(rng, L_end, kind):
        L += piece
        n_fixed, rows = stream.schedule(L, F, H, W, fps, first_row=len(got), **kw)
        assert n_fixed >= len(got), "rows are never withdrawn"
        assert n_fixed == _expected_fixed(L, fps, F, box is not None or nosmooth or F == 1), (L, n_fixed)
        M = _mel_final(L)
        for r in rows:
            assert r[0] == len(got), "gap-free, in order"
            assert r[1] + 16 <= M, "rule 2: the chunk is final and regular"
            got.append(tuple(int(v) for v in r))
    if ref is None:
        with pytest.raises(ValueError):
            stream.schedule(L_end, F, H, W, fps, final=True, **kw)
        assert not got
        return
    n_fixed, rows = stream.schedule(L_end, F, H, W, fps, final=True, first_row=len(got), **kw)
    assert n_fixed == len(ref)
    got += [tuple(int(v) for v in r) for r in rows]
    np.testing.assert_array_equal(np.asarray(got, dtype=np.int64).reshape(-1, 7), ref)


@pytest.mark.parametrize("L_end", [2, 399, 400, 401, 3399, 3400, 3401])
@pytest.mark.parametrize("fps", FPS)
@pytest.mark.parametrize("F", [1, 3, 7, 60])
def test_edge_lengths_one_sample_pushes(L_end, fps, F):
    for nosmooth, box in ((False, None), (True, None), (False, (5, 60, 7, 80))):
        _run(L_end, fps, F, nosmooth, box, "ones" if L_end <= 3401 else "random", seed=L_end + F)


@pytest.mark.parametrize("fps", FPS)
@pytest.mark.parametrize("F", [1, 3, 7, 60])
@pytest.mark.parametrize("kind", ["one", "640", "random"])
def test_random_lengths_and_splits(fps, F, kind):
    rng = np.random.default_rng(int(fps * 100) + F)
    for t in range(12):
        L_end = int(rng.integers(2, 16000 * 4))
        nosmooth = bool(t % 3 == 1)
        box = (3, 50, 10, 70) if t % 3 == 2 else None
        _run(L_end, fps, F, nosmooth, box, kind, seed=t)


def test_right_aligned_last_chunk_or_not():
    """The last chunk is always right-aligned (start M - 16 < s_i); lengths where it lands between two grid starts and
    lengths where it repeats the previous chunk (M - 16 == s_{i-1})."""
    seen = set()
    for L_end in range(3400, 3400 + 200 * 40, 200):
        for fps in FPS:
            ref = offline_rows(L_end, fps, 7, H, W, box=(0, 40, 0, 40))
            assert int(ref[-1][1]) == L_end // 200 + 1 - 16 < int(int(ref[-1][0]) * (80. / fps))
            seen.add(int(ref[-1][1]) == int(ref[-2][1]))
            _run(L_end, fps, 7, False, None, "640", seed=L_end)
    assert seen == {True, False}


def test_bad_arguments():
    with pytest.raises(Exception):
        stream.schedule(1000, 3, H, W, 0.0, box=(0, 10, 0, 10))
    with pytest.raises(Exception):
        stream.schedule(1000, 3, H, W, 25.0)                       # neither rects nor box
    with pytest.raises(ValueError):
        stream.schedule(1000, 3, H, W, 25.0, rects=np.zeros((2, 4)))


def test_rule1_against_the_reference_arithmetic():
    """The spectrum of wav[:L] (pre-emphasis, reflect padding, window, FFT: audio.py:45-47) equals the full wav's in every
    frame f with 200 f + 400 <= L, bit for bit, and so does the mel: everything after the FFT is per frame.  (NumPy's
    mel product is one BLAS matrix product over all frames, whose float32 rounding may depend on the frame count by an
    ulp; the kernel computes each frame on its own, so the column is compared after a per-frame product.)"""
    from oracle import mel_oracle as M
    wav = M.make_wav(6000, seed=3, kind="mix")

    def per_frame_mel(w):
        S = np.abs(M.stft(M.preemphasis(w)))
        cols = [M.linear_to_mel(S[:, f:f + 1]) for f in range(S.shape[1])]
        return S, M.normalize(M.amp_to_db(np.concatenate(cols, axis=1)) - np.float32(M.REF_LEVEL_DB))

    S_full, mel_full = per_frame_mel(wav)
    for L in (2, 399, 400, 401, 600, 799, 800, 1001, 3399, 3400, 3401, 5999):
        S, mel = per_frame_mel(wav[:L])
        f_final = _mel_final(L)
        np.testing.assert_array_equal(S[:, :f_final], S_full[:, :f_final])
        np.testing.assert_array_equal(mel[:, :f_final], mel_full[:, :f_final])
        if L >= 800:   # and the rule is tight: the next frame reflects at the prefix's end
            assert not np.array_equal(S[:, f_final], S_full[:, f_final])
    # the per-frame product is the oracle's mel up to that BLAS rounding
    np.testing.assert_allclose(mel_full, M.melspectrogram(wav), rtol=0, atol=2e-6)
