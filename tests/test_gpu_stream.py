"""Streaming on the GPU: `audio.MelStream` against `w2l_melspectrogram` on the whole wav, and `stream.LipSyncSession`
against the offline composition of inference.py (`audio.melspectrogram` -> `audio.mel_chunks` -> `face_boxes` on the
truncated rects -> `Wav2Lip.infer_frames`), bit for bit and frame for frame."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import mel_oracle as M
from oracle import w2l_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from stream_offline import random_rects  # noqa: E402

pytestmark = pytest.mark.gpu

EDGE = [2, 399, 400, 401, 3399, 3400, 3401]
H, W = 72, 88


def _splits(rng, n, kind):
    if kind == "one":
        return [n]
    if kind == "ones":
        return [1] * n
    if kind == "640":
        return [640] * (n // 640) + ([n % 640] if n % 640 else [])
    out, left = [], n
    while left:
        k = int(min(left, rng.integers(1, 5000)))
        out.append(k)
        left -= k
    return out


# ---------------------------------------------------------------------------------------------------------------------
# MelStream
# ---------------------------------------------------------------------------------------------------------------------
def _melstream(wav, splits, cuda_in, ring_log2=0):
    from wav2lip_b200 import audio
    ms = audio.MelStream(0, ring_log2)
    parts, at = [], 0
    src = torch.from_numpy(wav).cuda() if cuda_in else wav
    for k in splits:
        p = ms.push(src[at:at + k])
        at += k
        parts.append(p.cpu().numpy() if cuda_in else p)
    p = ms.finish()
    parts.append(p.cpu().numpy() if cuda_in else p)
    assert not ms.nan_seen()
    ms.close()
    return np.concatenate(parts, axis=1)


@pytest.mark.parametrize("n", EDGE + [48000 + 123])
@pytest.mark.parametrize("kind", ["one", "640", "random", "ones"])
def test_melstream_bit_identical(n, kind):
    from wav2lip_b200 import audio
    if kind == "ones" and n > 3401:
        pytest.skip("one-sample pushes on the short clips only")
    wav = M.make_wav(n, seed=n, kind="mix")
    ref = audio.melspectrogram(torch.from_numpy(wav).cuda()).cpu().numpy()
    rng = np.random.default_rng(n)
    for cuda_in in (False, True):
        got = _melstream(wav, _splits(rng, n, kind), cuda_in)
        assert got.shape == ref.shape
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_melstream_ten_minutes_smallest_ring_and_memory():
    """10 minutes through the 2^11-sample ring (it wraps ~4700 times); device memory after 1 s equals after 10 min."""
    from wav2lip_b200 import audio
    n = 16000 * 600 + 77
    wav = (0.1 * np.sin(np.arange(n) * 0.0123) + 0.01 * np.random.default_rng(0).standard_normal(n)).astype(np.float32)
    x = torch.from_numpy(wav).cuda()
    ref = audio.melspectrogram(x)
    ms = audio.MelStream(0, 11)
    ctx = audio._context(0)
    got, at, step, mem_1s = [], 0, 3001, None
    while at < n:
        got.append(ms.push(x[at:at + step]))
        at += step
        if mem_1s is None and at >= 16000:
            torch.cuda.synchronize()
            mem_1s = ctx.device_bytes()
    got.append(ms.finish())
    torch.cuda.synchronize()
    assert ctx.device_bytes() == mem_1s
    got = torch.cat(got, dim=1)
    assert got.shape == ref.shape
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))
    ms.close()


# ---------------------------------------------------------------------------------------------------------------------
# LipSyncSession
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gen():
    from wav2lip_b200.models import Wav2Lip
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
    return g.cuda().eval()


def _video(F, seed=0):
    rng = np.random.default_rng(seed)
    frames = torch.from_numpy(rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)).cuda()
    return frames, random_rects(rng, F, H, W)


def _offline(g, frames, wav, fps, rects=None, box=None, nosmooth=False, pads=(0, 10, 0, 0), batch=128):
    from wav2lip_b200 import audio
    from wav2lip_b200.face_detection import face_boxes
    mel = audio.melspectrogram(wav)
    chunks = torch.from_numpy(audio.mel_chunks(mel, fps)).cuda()
    n = chunks.shape[0]
    F = frames.shape[0]
    n_total = min(n, F)
    if box is not None:
        bx = np.asarray([box] * n_total, dtype=np.int64)
    else:
        bx = face_boxes([tuple(int(v) for v in r) for r in rects[:n_total]], H, W, pads, nosmooth)
    rows = np.asarray([(i % n_total,) + tuple(bx[i % n_total]) for i in range(n)], dtype=np.int32)
    with torch.no_grad():
        return torch.cat([g.infer_frames(chunks[k:k + batch], frames, rows[k:k + batch]) for k in range(0, n, batch)])


def _stream(g, frames, wav, fps, splits, batch, **kw):
    from wav2lip_b200.stream import LipSyncSession
    s = LipSyncSession(g, frames, fps, batch=batch, **kw)
    outs, at, expect = [], 0, 0
    for k in splits:
        first, fr = s.push(wav[at:at + k])
        at += k
        assert first == expect
        expect += fr.shape[0]
        outs.append(fr)
    first, fr = s.finish()
    assert first == expect
    outs.append(fr)
    s.close()
    return torch.cat(outs)


CASES = [  # (F, seconds of audio, fps, nosmooth, box, chunk count)
    (12, 0.30, 25.0, False, None, 5),           # audio shorter than the video
    (12, 0.60, 25.0, False, None, 12),          # equal: as many chunks as frames (9637 samples, 49 mel frames)
    (12, 1.30, 25.0, False, None, 30),          # longer
    (1, 0.70, 25.0, False, None, 15),           # a still image
    (12, 0.90, 29.97002997, True, None, 23),    # nosmooth
    (12, 0.90, 29.97002997, False, (5, 60, 7, 80), 23),   # a fixed box
]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("batch", [1, 4, 16])
@pytest.mark.parametrize("kind", ["640", "random"])
def test_session_matches_offline(gen, case, batch, kind):
    from wav2lip_b200 import audio
    F, sec, fps, nosmooth, box, n_chunks = CASES[case]
    frames, rects = _video(F, seed=case)
    n = int(sec * 16000) + 37 * case
    assert audio.num_chunks(audio.num_frames(n), fps) == n_chunks
    wav = M.make_wav(n, seed=case, kind="mix")
    kw = dict(rects=None if box else rects, box=box, nosmooth=nosmooth)
    got = _stream(gen, frames, wav, fps, _splits(np.random.default_rng(case + batch), n, kind), batch, **kw)
    ref = _offline(gen, frames, wav, fps, batch=batch, **kw)
    assert got.shape == ref.shape
    assert torch.equal(got, ref)
    # the offline run at batch 128 (dispatch choices that depend on N keep the K order, DESIGN.md section 3.1)
    assert torch.equal(got, _offline(gen, frames, wav, fps, batch=128, **kw))


def test_graph_on_and_off_identical(monkeypatch):
    from wav2lip_b200.models import Wav2Lip
    frames, rects = _video(12, seed=5)
    wav = M.make_wav(16000 + 321, seed=5, kind="mix")
    outs = []
    for off in ("0", "1"):
        monkeypatch.setenv("W2L_DISABLE_STREAMGRAPH", off)
        g = Wav2Lip()
        g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
        g = g.cuda().eval()
        outs.append(_stream(g, frames, wav, 25.0, [640] * 26, 4, rects=rects))
    assert torch.equal(outs[0], outs[1])


def test_new_weights_between_pushes():
    from wav2lip_b200.models import Wav2Lip
    from wav2lip_b200.stream import LipSyncSession
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
    g = g.cuda().eval()
    frames, rects = _video(40, seed=7)
    wav = M.make_wav(16000, seed=7, kind="mix")
    s = LipSyncSession(g, frames, 25.0, rects=rects, batch=4)
    outs = [s.push(wav[i * 640:(i + 1) * 640])[1] for i in range(12)]
    n_old = sum(o.shape[0] for o in outs)
    ref_old = _offline(g, frames, wav, 25.0, rects=rects, batch=4)
    g.load_state_dict(O.make_state_dict("generator", 1, init="default"), strict=True)
    outs += [s.push(wav[i * 640:(i + 1) * 640])[1] for i in range(12, 25)]
    outs.append(s.finish()[1])
    s.close()
    got = torch.cat(outs)
    ref_new = _offline(g, frames, wav, 25.0, rects=rects, batch=4)
    assert n_old > 0 and got.shape == ref_new.shape
    assert torch.equal(got[:n_old], ref_old[:n_old])
    assert torch.equal(got[n_old:], ref_new[n_old:])


def test_two_sessions_interleaved(gen):
    from wav2lip_b200.stream import LipSyncSession
    fa, ra = _video(12, seed=8)
    fb, rb = _video(5, seed=9)
    wa = M.make_wav(14000, seed=8, kind="mix")
    wb = M.make_wav(20000, seed=9, kind="noise")
    sa = LipSyncSession(gen, fa, 25.0, rects=ra, batch=4)
    sb = LipSyncSession(gen, fb, 29.97002997, rects=rb, batch=4)
    oa, ob = [], []
    for i in range(32):
        oa.append(sa.push(wa[i * 640:(i + 1) * 640])[1])
        ob.append(sb.push(wb[i * 640:(i + 1) * 640])[1])
    oa.append(sa.finish()[1])
    ob.append(sb.finish()[1])
    assert torch.equal(torch.cat(oa), _offline(gen, fa, wa, 25.0, rects=ra, batch=4))
    assert torch.equal(torch.cat(ob), _offline(gen, fb, wb, 29.97002997, rects=rb, batch=4))


def test_nan_mid_stream(gen):
    from wav2lip_b200.stream import LipSyncSession
    frames, rects = _video(60, seed=10)
    wav = M.make_wav(32000, seed=10, kind="mix")
    bad = wav.copy()
    bad[20000] = np.nan
    s = LipSyncSession(gen, frames, 25.0, rects=rects, batch=1)
    got, raised = [], None
    for i in range(50):
        try:
            got.append(s.push(bad[i * 640:(i + 1) * 640])[1])
        except ValueError as e:
            raised = (i, str(e))
            break
    assert raised is not None and raised[1].startswith("Mel contains nan! Using a TTS voice?")
    # raised by the push that computes the first NaN frame: frame 99 reads pre-emphasised samples [19400, 20200), and
    # samples 20000 and 20001 are NaN after pre-emphasis; it is final once 200 * 99 + 400 = 20200 samples have arrived,
    # in push 31 (samples 19840 .. 20479)
    assert raised[0] == 31
    with pytest.raises(ValueError, match="Mel contains nan!"):
        s.finish()
    got = torch.cat(got)
    # every returned frame is the offline frame of the same audio without the NaN (its chunk does not reach sample 20000)
    clean = _offline(gen, frames, wav, 25.0, rects=rects, batch=1)
    assert torch.equal(got, clean[:got.shape[0]])
    last_frame = int((got.shape[0] - 1) * (80. / 25.0)) + 15       # last mel frame of the last returned chunk
    assert 200 * last_frame + 400 <= 20000                          # it read samples before the NaN only
    s.close()


def test_pinned_plan_survives_lru_eviction(gen):
    """Between two pushes of a live session, other batch sizes build and evict plans (at most 6 per net stay): the
    session's graph replays its own plan, which the eviction must skip, and its output still equals the offline run."""
    from wav2lip_b200.stream import LipSyncSession
    frames, rects = _video(12, seed=12)
    wav = M.make_wav(24000, seed=12, kind="mix")
    s = LipSyncSession(gen, frames, 25.0, rects=rects, batch=4)
    outs = [s.push(wav[i * 640:(i + 1) * 640])[1] for i in range(14)]     # the graph is captured by now
    chunks = torch.rand(9, 1, 80, 16, device="cuda")
    rows = np.asarray([(j % 12, 5, 60, 7, 80) for j in range(9)], dtype=np.int32)
    with torch.no_grad():
        for N in (1, 2, 3, 5, 6, 7, 8, 9):                # eight other plans: more than the LRU keeps
            gen.infer_frames(chunks[:N], frames, rows[:N])
    outs += [s.push(wav[i * 640:(i + 1) * 640])[1] for i in range(14, 38)]    # the last piece is 320 samples
    outs.append(s.finish()[1])
    s.close()
    assert torch.equal(torch.cat(outs), _offline(gen, frames, wav, 25.0, rects=rects, batch=4))


def test_bad_arguments(gen):
    import ctypes as C

    from wav2lip_b200 import _lib, stream
    from wav2lip_b200.stream import LipSyncSession
    frames, rects = _video(6, seed=11)
    launches = gen._w2l_ctx.launch_count() if gen._w2l_ctx else None
    with pytest.raises(_lib.W2LError):
        LipSyncSession(gen, frames.cpu(), 25.0, rects=rects)
    with pytest.raises(ValueError):
        LipSyncSession(gen, frames, 25.0, rects=rects[:4])
    with pytest.raises(ValueError):
        LipSyncSession(gen, frames, 25.0, rects=rects, batch=0)
    with pytest.raises(ValueError):
        LipSyncSession(gen, frames, 0.0, rects=rects)
    with pytest.raises(ValueError):
        LipSyncSession(gen, frames, 25.0)
    # a frame of 2^31 bytes or more (the paste's offsets within a frame are 32-bit), described over a small real video
    ctx = gen._ensure(frames)
    big = stream._desc(1, 1, 2 ** 31 // 3 + 1, 25.0, (0, 10, 0, 0), False, (0, 1, 0, 1))
    h = C.c_void_p()
    with pytest.raises(_lib.W2LError, match=r"2\^31"):
        _lib.check(ctx.lib.w2l_stream_create(ctx.h, C.c_void_p(frames.data_ptr()), C.byref(big), None, 1, C.byref(h)))
    if launches is not None:
        assert gen._w2l_ctx.launch_count() == launches
