"""Training data pipeline on the GPU (wav2lip_b200/data.py, csrc/train_data.cuh): the device cache and the two gather kernels
write exactly what `default_collate` of the reference Datasets' `__getitem__` calls returns.

* golden: batches from `TrainDataCache.from_arrays(fixture)` hash to the sha256 the reference produced
  (tests/golden/train_data.npz), both datasets, B = 1, 4 and 16 (hparams.batch_size; 10 videos, so one short batch);
* B = 64 over a random 2 000-frame cache holding all 256 byte values: bit for bit against the NumPy restatement
  (tests/train_data_restated.py), which divides by 255 in float64 as NumPy does;
* pinned storage gives the same bytes as device storage; two runs are identical;
* a cache built from wavs holds mels within the mel bar (1e-4) of the oracle;
* bad sample tables and pageable pointers raise W2LError with nothing launched;
* one `Wav2LipTrainStep` on an assembled batch equals the step on the same batch built on the host and copied."""
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import train_data_restated as R  # noqa: E402

from wav2lip_b200 import _lib, audio  # noqa: E402
from wav2lip_b200 import data as D  # noqa: E402

pytestmark = pytest.mark.gpu
SEEDS = (0, 1, 7)


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "train_data.npz"))


@pytest.fixture(scope="module")
def fixture_cache(gold):
    return D.TrainDataCache.from_arrays(R.fixture_videos(gold))


def _random_videos(seed, n_videos=40, n_frames=50, n_mel=160):
    rng = np.random.default_rng(seed)
    vids = []
    for i in range(n_videos):
        names = [f"{k}.jpg" for k in rng.permutation(n_frames)]
        crops = list(rng.integers(0, 256, (n_frames, 96, 96, 3), dtype=np.uint8))
        crops[0][0, 0, 0], crops[0][0, 1, 0] = 0, 255
        crops[int(rng.integers(1, n_frames))] = None if i % 7 == 3 else crops[1]
        mel = rng.standard_normal((n_mel + i, 80)).astype(np.float32) * 4
        vids.append({"img_names": names, "crops": crops, "mel": mel})
    return vids


@pytest.fixture(scope="module")
def random_cache():
    vids = _random_videos(5)
    cache = D.TrainDataCache.from_arrays(vids)
    frames = cache.frames.cpu().numpy()
    assert len(np.unique(frames)) == 256
    return vids, cache, frames, cache.mels.cpu().numpy()


def _np(ts):
    return [t.cpu().numpy() for t in ts]


@pytest.mark.parametrize("tag", ["w2l", "sync"])
@pytest.mark.parametrize("seed", SEEDS)
def test_device_batches_match_reference_hashes(gold, fixture_cache, tag, seed):
    cls = D.Wav2LipBatches if tag == "w2l" else D.SyncNetBatches
    for B in (1, 4, 16):
        got = [[R.sha(t) for t in _np(batch)] for batch in cls(fixture_cache, B, rng=random.Random(seed)).epoch()]
        assert np.array_equal(np.array(got), gold[f"{tag}_s{seed}_b{B}_sha"]), (tag, seed, B)


def test_fixture_cache_frames_are_cv2_resized(gold, fixture_cache):
    frames, mels = R.cache_arrays(R.fixture_videos(gold))
    readable = np.array([c is not None for v in R.fixture_videos(gold) for c in v["crops"]])
    assert np.array_equal(fixture_cache.frames.cpu().numpy()[readable], frames[readable])
    assert np.array_equal(fixture_cache.mels.cpu().numpy(), mels)


@pytest.mark.parametrize("tag", ["w2l", "sync"])
def test_b64_bit_exact_against_numpy(random_cache, tag):
    _, cache, frames, mels = random_cache
    cls, build = (D.Wav2LipBatches, R.wav2lip_batch) if tag == "w2l" else (D.SyncNetBatches, R.syncnet_batch)
    b = cls(cache, 64, rng=random.Random(11))
    for _ in range(3):
        table = b.samples(64)
        got = _np(b.assemble(table))
        want = build(frames, mels, table.tolist())
        for g, w in zip(got, want):
            assert g.shape == w.shape and g.dtype == w.dtype
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32))
    # every byte value reaches the output through the table (u * (1/255.f) differs on 126 of them)
    lut = (np.arange(256) / 255.).astype(np.float32)
    assert (lut != np.arange(256, dtype=np.float32) * np.float32(1 / 255.)).sum() == 126
    table = np.array([[s] * 5 + ([s] * 5 + [0] * 6 if tag == "w2l" else [0, 1]) + [cache.videos[0].mel_len]
                      for s in range(64)], dtype=np.int32)
    x = _np(b.assemble(table))[0]
    vals = np.unique(x[:, 3:6] if tag == "w2l" else x)
    assert set(np.unique(frames[:64, 48:] if tag == "sync" else frames[:64]).tolist()) == \
        set(np.rint(vals * 255).astype(int).tolist())
    assert np.array_equal(np.sort(vals), np.sort(lut[np.rint(vals * 255).astype(int)]))


def test_pinned_storage_gives_device_bytes(random_cache):
    vids, cache, frames, _ = random_cache
    pinned = D.TrainDataCache.from_arrays(vids, storage="pinned")
    assert not pinned.frames.is_cuda and pinned.frames.is_pinned()
    assert np.array_equal(pinned.frames.numpy(), frames)
    for cls in (D.Wav2LipBatches, D.SyncNetBatches):
        table = cls(cache, 64, rng=random.Random(3)).samples(64)
        a = _np(cls(cache, 64).assemble(table))
        p = _np(cls(pinned, 64).assemble(table))
        for u, v in zip(a, p):
            assert np.array_equal(u.view(np.uint32), v.view(np.uint32))


def test_two_runs_identical(random_cache):
    _, cache, _, _ = random_cache
    for cls in (D.Wav2LipBatches, D.SyncNetBatches):
        r1 = [_np(t) for t in cls(cache, 16, rng=random.Random(9)).epoch()]
        r2 = [_np(t) for t in cls(cache, 16, rng=random.Random(9)).epoch()]
        assert len(r1) == 3 and r1[-1][0].shape[0] == 40 - 32
        for a, b in zip(r1, r2):
            for u, v in zip(a, b):
                assert np.array_equal(u.view(np.uint32), v.view(np.uint32))


def test_cache_from_wavs_holds_device_mels():
    from oracle import mel_oracle as M
    wavs = [M.make_wav(n, seed=20 + n % 7, kind="mix") for n in (8000, 12345, 16000)]
    vids = [{"img_names": [f"{k}.jpg" for k in range(3)], "crops": [np.zeros((50, 60, 3), np.uint8)] * 3, "wav": w}
            for w in wavs]
    vids.append({"img_names": ["0.jpg"], "crops": [np.zeros((8, 8, 3), np.uint8)], "wav": None})
    cache = D.TrainDataCache.from_arrays(vids)
    mels = cache.mels.cpu().numpy()
    for v, w in zip(cache.videos, wavs):
        ref = M.melspectrogram(w).T
        assert v.mel_len == ref.shape[0]
        assert float(np.abs(mels[v.mel_off:v.mel_off + v.mel_len] - ref).max()) <= 1e-4
    assert cache.videos[-1].mel_len == -1


def test_bad_tables_and_pageable_memory_launch_nothing(random_cache):
    _, cache, _, _ = random_cache
    ctx = audio._context(cache.device.index)
    b = D.Wav2LipBatches(cache, 4, rng=random.Random(1))
    good = b.samples(4)
    n0 = ctx.launch_count()
    bad_cases = []
    for k, v in ((0, cache.n_frames), (7, -1), (10, cache.n_mel_rows), (13, cache.n_mel_rows - 8), (16, cache.n_mel_rows + 1)):
        t = good.copy()
        t[2, k] = v
        bad_cases.append(t)
    for t in bad_cases:
        with pytest.raises(_lib.W2LError):
            b.assemble(t)
    s = D.SyncNetBatches(cache, 4, rng=random.Random(1))
    t = s.samples(4)
    t[1, 6] = 3
    with pytest.raises(_lib.W2LError, match="label 3"):
        s.assemble(t)
    host = D.TrainDataCache(cache.videos, cache.frames.cpu(), cache.mels, cache.device)         # pageable frames
    with pytest.raises(_lib.W2LError, match="frames is pageable"):
        D.Wav2LipBatches(host, 4).assemble(good)
    host = D.TrainDataCache(cache.videos, cache.frames, cache.mels.cpu(), cache.device)         # pageable mels
    with pytest.raises(_lib.W2LError, match="mels is pageable"):
        D.SyncNetBatches(host, 4).assemble(s.samples(4))
    torch.cuda.synchronize()
    assert ctx.launch_count() == n0
    b.assemble(good)
    assert ctx.launch_count() == n0 + 1


def test_train_step_on_assembled_batch_equals_host_batch(random_cache):
    from wav2lip_b200.models import SyncNet_color, Wav2Lip
    from wav2lip_b200.training import Wav2LipTrainStep
    _, cache, frames, mels = random_cache
    b = D.Wav2LipBatches(cache, 4, rng=random.Random(2))
    table = b.samples(4)
    dev_batch = b.assemble(table)
    host_batch = [torch.from_numpy(a).cuda() for a in R.wav2lip_batch(frames, mels, table.tolist())]
    results = []
    for batch in (dev_batch, host_batch):
        torch.manual_seed(0)
        gen, expert = Wav2Lip().cuda().train(), SyncNet_color().cuda().train()
        step = Wav2LipTrainStep(gen, expert, lr=1e-4, syncnet_wt=0.03)
        losses = step(*batch).cpu().numpy()
        torch.cuda.synchronize()
        results.append((losses, {k: v.detach().cpu().clone() for k, v in gen.state_dict().items()}))
    assert np.array_equal(results[0][0], results[1][0])
    for k, v in results[0][1].items():
        assert torch.equal(v, results[1][1][k]), k
