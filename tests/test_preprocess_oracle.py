"""oracle/preprocess_oracle.py against the real preprocess.py (tests/golden/preprocess.npz, made by
tests/golden/make_golden_preprocess.py): for every scripted video, the files it leaves, whether it was abandoned, and each
crop's shape and bytes; and `data.write_face_crops` on the oracle's rows writes the script's jpg bytes."""
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import preprocess_oracle as P  # noqa: E402

G = np.load(os.path.join(ROOT, "tests", "golden", "preprocess.npz"))
CASES = list(G["case_names"])


def _case(k):
    frames, has, dets = G[f"c{k}_frames"], G[f"c{k}_has"], G[f"c{k}_dets"]
    return frames, [dets[f] if has[f] else None for f in range(len(has))], int(G[f"c{k}_batch"])


@pytest.mark.parametrize("k", range(len(CASES)), ids=CASES)
def test_oracle_matches_the_script(k):
    frames, dets, batch = _case(k)
    rows = P.preprocess_rows(dets, frames.shape[1], frames.shape[2], batch)
    assert rows.dtype == np.int32 and rows.shape == (len(dets), 6)
    assert P.files(rows) == list(G[f"c{k}_files"])
    assert P.aborted(rows) == bool(G[f"c{k}_aborted"])
    cr = P.crops(frames, rows)
    assert [list(c.shape) for c in cr] == G[f"c{k}_shapes"].tolist()
    assert [hashlib.sha256(np.ascontiguousarray(c).tobytes()).hexdigest() for c in cr] == list(G[f"c{k}_sha_arr"])
    # slots are dealt in frame order; every lost frame follows the abort point
    kept = rows[:, 0] == P.KEPT
    assert rows[kept, 1].tolist() == list(range(int(kept.sum())))
    assert (rows[~kept, 1] == -1).all()
    lost = np.flatnonzero(rows[:, 0] == P.ABORTED)
    if len(lost):
        cause = np.flatnonzero((rows[:, 0] == P.NON_FINITE) | (rows[:, 0] == P.EMPTY))
        assert len(cause) == 1 and (lost > cause[0] - batch).all()


def test_cases_cover_the_rules():
    status = set()
    for k in range(len(CASES)):
        frames, dets, batch = _case(k)
        status |= set(P.preprocess_rows(dets, frames.shape[1], frames.shape[2], batch)[:, 0].tolist())
    assert status == {P.KEPT, P.NO_FACE, P.NON_FINITE, P.EMPTY, P.ABORTED}


def test_box_rules():
    H, W = 64, 80
    assert P.frame_box(None, H, W) == (P.NO_FACE, (0, 0, 0, 0))
    assert P.frame_box([-np.inf, -2.5, 1e30, 10.99], H, W) == (P.KEPT, (0, 10, 0, W))
    assert P.frame_box([np.nan, 1, 2, 3], H, W)[0] == P.NON_FINITE
    assert P.frame_box([1, 2, np.inf, 3], H, W)[0] == P.NON_FINITE
    assert P.frame_box([W, 0, W + 5, 10], H, W)[0] == P.EMPTY
    # a NaN in the first batch loses the whole batch, the empty crop after it is not the cause
    rows = P.preprocess_rows([[1, 1, 9, 9]] * 2 + [[1, 1, 1, 9], [np.nan, 1, 9, 9], [1, 1, 9, 9]], H, W, batch=4)
    assert rows[:, 0].tolist() == [4, 4, 4, 2, 4]
    rows = P.preprocess_rows([[1, 1, 9, 9]] * 2 + [[1, 1, 1, 9], [np.nan, 1, 9, 9], [1, 1, 9, 9]], H, W, batch=3)
    assert rows[:, 0].tolist() == [0, 0, 3, 4, 4]


@pytest.mark.parametrize("k", range(len(CASES)), ids=CASES)
def test_write_face_crops_writes_the_script_files(k, tmp_path):
    cv2 = pytest.importorskip("cv2")
    from wav2lip_b200.data import write_face_crops
    frames, dets, batch = _case(k)
    rows = P.preprocess_rows(dets, frames.shape[1], frames.shape[2], batch)
    d = str(tmp_path / "vid")
    names = write_face_crops(d, frames, rows)
    assert names == list(G[f"c{k}_files"])
    assert sorted(os.listdir(d)) == sorted(names) if names else not os.path.exists(d) or os.listdir(d) == []
    if cv2.__version__ != str(G["cv2_version"]):
        pytest.skip(f"jpg bytes pinned with OpenCV {G['cv2_version']}, this is {cv2.__version__}")
    got = [hashlib.sha256(open(os.path.join(d, n), "rb").read()).hexdigest() for n in names]
    assert got == list(G[f"c{k}_sha_jpg"])
