"""audio.melspectrogram on the GPU (C-ABI w2l_melspectrogram[_host]) against the oracle and its
committed vectors; tolerance 1e-4 (north_star).  The librosa boundary is unpinned — see
oracle/mel_oracle.py."""
import os

import numpy as np
import pytest
import torch

from oracle import mel_oracle as M

pytestmark = pytest.mark.gpu

TOL = 1e-4


@pytest.mark.parametrize("kind", ["noise", "sweep", "mix"])
def test_mel_golden(kind, golden_dir):
    from wav2lip_b200 import audio
    g = np.load(os.path.join(golden_dir, "mel.npz"))
    wav = M.make_wav(48000 + 137, seed=7, kind=kind)
    mel = audio.melspectrogram(wav)
    assert mel.dtype == np.float32 and mel.shape == g["mel_" + kind].shape
    assert np.abs(mel - g["mel_" + kind]).max() <= TOL
    assert mel.min() >= -4.0 and mel.max() <= 4.0


def test_mel_config3_10k_frames():
    """BASELINE configs[2]: 1 999 800 samples -> exactly 10 000 frames, whole array against the oracle."""
    from wav2lip_b200 import audio
    wav = M.make_wav(1999800, seed=11, kind="mix")
    ref = M.melspectrogram(wav)
    mel = audio.melspectrogram(wav)
    assert mel.shape == (80, 10000)
    assert np.abs(mel - ref).max() <= TOL


def test_mel_device_tensor_path_and_edges():
    from wav2lip_b200 import _lib, audio
    wav = M.make_wav(16000, seed=2, kind="sweep")
    m_host = audio.melspectrogram(wav)
    m_dev = audio.melspectrogram(torch.from_numpy(wav).cuda())
    assert m_dev.is_cuda and np.array_equal(m_dev.cpu().numpy(), m_host)
    wav = M.make_wav(16000 * 4 + 321, seed=13, kind="mix")
    assert np.abs(audio.melspectrogram(torch.from_numpy(wav).cuda()).cpu().numpy() - M.melspectrogram(wav)).max() <= TOL
    # silence -> the 1e-5 floor -> exactly -4.0
    z = audio.melspectrogram(np.zeros(4000, dtype=np.float32))
    assert z.shape == (80, 21) and np.all(z == -4.0)
    s = audio.melspectrogram(np.ones(401, dtype=np.float32))
    assert s.shape == (80, 3) and np.abs(s - M.melspectrogram(np.ones(401, dtype=np.float32))).max() <= TOL
    # clips shorter than n_fft/2: np.pad(mode="reflect") folds the index more than once (librosa 0.7.0 does not check)
    for L in (400, 399, 201, 200, 57, 2):
        w = M.make_wav(L, seed=100 + L, kind="noise")
        got = audio.melspectrogram(w)
        assert got.shape == (80, 1 + L // 200) and np.abs(got - M.melspectrogram(w)).max() <= TOL, L
    with pytest.raises(_lib.W2LError):
        audio.melspectrogram(np.ones(1, dtype=np.float32))
    # lengths around hop / block boundaries
    for L in (801, 999, 1000, 1001, 1599, 1600, 3217):
        w = M.make_wav(L, seed=L, kind="noise")
        assert np.abs(audio.melspectrogram(w) - M.melspectrogram(w)).max() <= TOL, L


def test_mel_loud_tone_near_floor():
    """A loud pure tone puts most bands ~100 dB below the peak, next to the clipping floor: the case
    a float32 FFT fails and the reason the kernel's FFT is float64."""
    from wav2lip_b200 import audio
    t = np.arange(32000) / 16000.0
    wav = (0.9 * np.sin(2 * np.pi * 1000.0 * t)).astype(np.float32)
    ref = M.melspectrogram(wav)
    assert np.abs(audio.melspectrogram(wav) - ref).max() <= TOL


def test_mel_shift_property():
    """Frames are independent given their 800 samples: mel(wav[200k:]) == mel(wav)[:, k:] away from the
    reflected edges, bit-exactly."""
    from wav2lip_b200 import audio
    wav = M.make_wav(40000, seed=5, kind="noise")
    a = audio.melspectrogram(wav)
    b = audio.melspectrogram(wav[2000:])
    # pre-emphasis makes sample 0 special and reflect padding touches 2 frames each side
    assert np.array_equal(a[:, 10 + 3:-3], b[:, 3:-3])

