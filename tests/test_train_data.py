"""Training data pipeline, host side (wav2lip_b200/data.py): the samplers replay the reference Datasets' `random` draws call for
call, the tensors they select reproduce the reference's bytes, the directory scan and decode match glob / cv2, and the C entry
points refuse bad sample tables before touching a device.

Golden data: tests/golden/train_data.npz (tests/golden/make_golden_train_data.py, from the reference's wav2lip_train.py and
color_syncnet_train.py run on a generated dataset with a ≤ 15-frame video, a missing id, a zero-byte jpg, a video without audio,
a short wav and crops of several shapes)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_data_restated as R  # noqa: E402

from wav2lip_b200 import data as D  # noqa: E402

SEEDS = (0, 1, 7)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "train_data.npz"))


@pytest.fixture(scope="module")
def videos(gold):
    return R.fixture_videos(gold)


@pytest.fixture(scope="module")
def arrays(videos):
    return R.cache_arrays(videos)


def _epoch_rows(index, sampler, seed):
    rng = R.LogRandom(seed)
    return [sampler(index, rng) for _ in range(len(index))], rng.log


def test_fixture_covers_the_rejection_cases(gold, videos):
    lens = [len(v["img_names"]) for v in videos]
    assert min(lens) <= 15
    assert any(c is None for v in videos for c in v["crops"])                      # zero-byte jpg
    assert any("mel" not in v for v in videos)                                     # no audio.wav
    assert any(len(v["img_names"]) > 15 and "7.jpg" not in v["img_names"] for v in videos)   # a gap
    shapes = {c.shape[:2] for v in videos for c in v["crops"] if c is not None}
    assert (96, 96) in shapes and any(h > 96 for h, _ in shapes) and any(h < 96 for h, _ in shapes)
    assert any(h != w for h, w in shapes)


@pytest.mark.parametrize("tag", ["w2l", "sync"])
@pytest.mark.parametrize("seed", SEEDS)
def test_sampler_replays_the_reference_draws(gold, videos, tag, seed):
    index = R.fixture_index(videos)
    sampler = D.sample_wav2lip if tag == "w2l" else D.sample_syncnet
    rows, log = _epoch_rows(index, sampler, seed)
    assert np.array_equal(np.array(log, dtype=np.int64), gold[f"{tag}_s{seed}_log"])
    for row, (vid, img, wrong, label) in zip(rows, gold[f"{tag}_s{seed}_picks"]):
        v, names = index[vid], videos[vid]["img_names"]
        fid = int(names[img].split(".")[0])
        off = v.mel_off
        if tag == "w2l":
            wid = int(names[wrong].split(".")[0])
            assert row[0:5] == [v.slots[f"{fid + t}.jpg"] for t in range(5)]
            assert row[5:10] == [v.slots[f"{wid + t}.jpg"] for t in range(5)]
            assert row[10] == off + (80 * fid) // 25
            assert row[11:16] == [off + (80 * (fid - 1 + k)) // 25 for k in range(5)]    # indiv mels start at id - 1
            assert row[16] == off + v.mel_len
        else:
            chosen = fid if label == 1 else int(names[wrong].split(".")[0])
            assert row[0:5] == [v.slots[f"{chosen + t}.jpg"] for t in range(5)]
            assert row[5] == off + (80 * fid) // 25                  # cut at img_name even when y = 0 (:118)
            assert row[6:8] == [label, off + v.mel_len]


def test_mel_start_matches_integer_form():
    n = np.arange(200000)
    assert all(D._mel_start(int(k)) == (80 * int(k)) // 25 for k in n[::997])
    assert [D._mel_start(k) for k in range(2000)] == [(80 * k) // 25 for k in range(2000)]


@pytest.mark.parametrize("tag", ["w2l", "sync"])
@pytest.mark.parametrize("seed", SEEDS)
def test_numpy_assembly_reproduces_golden_hashes(gold, videos, arrays, tag, seed):
    frames, mels = arrays
    index = R.fixture_index(videos)
    sampler = D.sample_wav2lip if tag == "w2l" else D.sample_syncnet
    build = R.wav2lip_batch if tag == "w2l" else R.syncnet_batch
    rows, _ = _epoch_rows(index, sampler, seed)
    for B in (1, 4, 16):
        want = gold[f"{tag}_s{seed}_b{B}_sha"]
        got = [[R.sha(t) for t in build(frames, mels, rows[i:i + B])] for i in range(0, len(rows), B)]
        assert np.array_equal(np.array(got), want), (tag, seed, B)


def test_wav2lip_sampler_rejects_frame_id_zero():
    """get_segmented_mels returns None at id 0 (start_frame_num - 2 < 0).  Here the only complete windows start at 0 and 30, and
    30's mel window is short, so every draw is rejected; SyncNet (no indiv mels) accepts id 0."""
    import random
    names = [f"{i}.jpg" for i in list(range(5)) + list(range(30, 35)) + list(range(10, 24, 2))]
    v = D.VideoIndex("v", names, range(len(names)), 0, 50)
    with pytest.raises(_Exhausted):
        D.sample_wav2lip([v], _Limited(random.Random(3), 5000))
    assert D.sample_syncnet([v], random.Random(3))[0:5] in ([0, 1, 2, 3, 4], [5, 6, 7, 8, 9])


class _Exhausted(Exception):
    pass


class _Limited:
    def __init__(self, rng, n):
        self.rng, self.n = rng, n

    def _tick(self):
        self.n -= 1
        if self.n < 0:
            raise _Exhausted

    def randint(self, a, b):
        self._tick()
        return self.rng.randint(a, b)

    def choice(self, seq):
        self._tick()
        return self.rng.choice(seq)


def test_get_image_list_reads_filelist_relative_to_cwd(tmp_path, monkeypatch):
    os.makedirs(tmp_path / "filelists")
    (tmp_path / "filelists" / "val.txt").write_text("a/b extra\nc\n")
    (tmp_path / "other.txt").write_text("d\n")
    monkeypatch.chdir(tmp_path)
    assert D.get_image_list("root", "val") == [os.path.join("root", "a/b"), os.path.join("root", "c")]
    assert D.get_image_list("root", "val", filelist=str(tmp_path / "other.txt")) == [os.path.join("root", "d")]


def test_scan_and_decode_match_glob_and_flags(gold, videos, tmp_path, monkeypatch):
    cv2 = pytest.importorskip("cv2")
    from glob import glob

    from scipy.io import wavfile
    root = tmp_path / "data"
    for i, v in enumerate(videos):
        d = root / f"vid{i:02d}"
        os.makedirs(d)
        for n, c in zip(v["img_names"], v["crops"]):
            (d / n).write_bytes(b"" if c is None else cv2.imencode(".png", c)[1].tobytes())
        if "mel" in v:
            wavfile.write(str(d / "audio.wav"), 16000, np.zeros(1600, np.int16))
    os.makedirs(tmp_path / "filelists")
    (tmp_path / "filelists" / "train.txt").write_text("".join(f"vid{i:02d}\n" for i in range(len(videos))))
    monkeypatch.chdir(tmp_path)
    scan = D.scan_data_root(str(root), "train")
    assert [p for p, _ in scan] == [os.path.join(str(root), f"vid{i:02d}") for i in range(len(videos))]
    for (vid, names), v in zip(scan, videos):
        assert names == [os.path.basename(p) for p in glob(os.path.join(vid, "*.jpg"))]
        assert sorted(names) == sorted(v["img_names"])
        dec = D.decode_video(vid, names)
        want = dict(zip(v["img_names"], v["crops"]))
        for n, c in zip(names, dec["crops"]):
            assert (c is None) == (want[n] is None), n
            if c is not None:
                assert np.array_equal(c, want[n])
        assert (dec["wav"] is None) == ("mel" not in v)


@pytest.fixture(scope="module")
def lib():
    from wav2lip_b200 import _lib
    if not os.path.exists(_lib.lib_path()):
        import __graft_entry__ as g
        g.build()
    return _lib


def _call(lib, tag, table, n_frames=100, n_mel_rows=500):
    L = lib.get_lib()
    t = np.ascontiguousarray(table, dtype=np.int32)
    p = C.c_void_p(1 << 20)           # never dereferenced: the table is refused before any pointer is used
    outs = [p] * (4 if tag == "w2l" else 3)
    fn = L.w2l_train_batch_wav2lip if tag == "w2l" else L.w2l_train_batch_syncnet
    r = fn(None, p, n_frames, p, n_mel_rows, t.ctypes.data_as(C.POINTER(C.c_int32)), t.shape[0], *outs, None)
    return r, L.w2l_last_error().decode()


def test_sample_table_validation_messages(lib):
    ok_w = [0, 1, 2, 3, 4, 10, 11, 12, 13, 14, 20, 17, 20, 23, 26, 29, 100]
    ok_s = [0, 1, 2, 3, 4, 20, 1, 100]
    assert _call(lib, "w2l", [ok_w]) == (lib.W2L_EINVAL, "null context")
    assert _call(lib, "sync", [ok_s]) == (lib.W2L_EINVAL, "null context")
    cases = [
        ("w2l", 3, 100, "sample 1: frame slot 100 is outside the 100 cached frames"),
        ("w2l", 7, -1, "sample 1: frame slot -1 is outside the 100 cached frames"),
        ("w2l", 16, 501, "sample 1: video end row 501 is past the 500 cached mel rows"),
        ("w2l", 10, 85, "sample 1: mel window at row 85 does not end by its video's end row 100"),
        ("w2l", 15, 90, "sample 1: mel window at row 90 does not end by its video's end row 100"),
        ("w2l", 11, -3, "sample 1: mel window at row -3 does not end by its video's end row 100"),
        ("sync", 4, 100, "sample 1: frame slot 100 is outside the 100 cached frames"),
        ("sync", 5, 85, "sample 1: mel window at row 85 does not end by its video's end row 100"),
        ("sync", 6, 2, "sample 1: label 2 is not 0 or 1"),
        ("sync", 7, 600, "sample 1: video end row 600 is past the 500 cached mel rows"),
    ]
    for tag, k, v, msg in cases:
        ok = ok_w if tag == "w2l" else ok_s
        bad = list(ok)
        bad[k] = v
        assert _call(lib, tag, [ok, bad]) == (lib.W2L_EINVAL, msg), (tag, k, v)
    r, msg = _call(lib, "w2l", [ok_w], n_mel_rows=8)
    assert r == lib.W2L_EINVAL and "mel rows" in msg
