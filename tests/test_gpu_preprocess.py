"""preprocess.py on the device: `w2l_face_crops_u8` against oracle/preprocess_oracle.py (pinned to the real script by
tests/golden/preprocess.npz) and oracle/pipeline_oracle.py's cv2-exact resize, and `face_crops` / `TrainDataCache.from_videos`
end to end with the device detector.

1. Kernel vs oracle: the golden's scripted detections uploaded as device dets / counts; rows equal the oracle's, every kept
   crop equals resize_linear_u8 of its slice bit for bit; under several call splits of each video (one call per detector
   batch, calls of 2·batch frames with a last call of up to 2·batch + 3, the whole video at once, one frame per call at
   batch 1); constructed edge boxes at 1280x720 and 1920x1080 (coordinates of 1e30, -inf, crops larger than 96 both ways);
   invalid arguments and the cap overflow.
2. End to end: seeded S3FD weights with a raised background bias, at 160x160 and 1280x720, with a bias chosen so that the
   video has frames with and without a face; face_crops' rows equal the oracle on the detector's own top boxes,
   from_videos equals from_arrays built from the host slices (frames bit for bit, index, mels), and the batch samplers
   return identical batches; pinned storage, and a video at 48 kHz.
"""
import ctypes as C
import os
import random

import numpy as np
import pytest
import torch

from oracle import pipeline_oracle as PO
from oracle import preprocess_oracle as P
from oracle import s3fd_oracle as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "preprocess.npz"))
CASES = list(G["case_names"])
TAPS = ["conv3_3_norm", "conv4_3_norm", "conv5_3_norm", "fc7", "conv6_2", "conv7_2"]


def _ctx():
    from wav2lip_b200 import audio
    return audio._context(torch.cuda.current_device())


def _p(t):
    return C.c_void_p(t.data_ptr())


def _run(frames_d, dets_d, counts_d, batch, calls, cap=None, out=None):
    """w2l_face_crops_u8 over one video in calls of the given sizes -> rows, state (host), crops (device)."""
    from wav2lip_b200 import _lib
    ctx = _ctx()
    F, H, W, _ = frames_d.shape
    out = torch.zeros((F, 96, 96, 3), dtype=torch.uint8, device="cuda") if out is None else out
    cap = out.shape[0] if cap is None else cap
    rows = torch.full((F, 6), -7, dtype=torch.int32, device="cuda")
    state = torch.zeros(2, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    s = 0
    for n in calls:
        _lib.check(ctx.lib.w2l_face_crops_u8(ctx.h, _p(frames_d[s:]), n, H, W, _p(dets_d[s:]), _p(counts_d[s:]),
                                             dets_d.shape[1], s, batch, _p(state), _p(rows[s:]), _p(out), cap, C.c_void_p(st)))
        s += n
    assert s == F
    torch.cuda.synchronize()
    return rows.cpu().numpy(), state.cpu().numpy(), out


def _splits(F, batch):
    out = {"whole": [F], "per_batch": [min(batch, F - s) for s in range(0, F, batch)]}
    calls, s = [], 0
    while F - s > 2 * batch + 3:
        calls.append(2 * batch)
        s += 2 * batch
    out["two_batches_last_up_to_2b3"] = calls + [F - s]
    return out


def _check(frames, dets, batch, rows, state, crops):
    H, W = frames.shape[1:3]
    want = P.preprocess_rows(dets, H, W, batch)
    assert np.array_equal(rows, want), np.flatnonzero((rows != want).any(axis=1))
    kept = int((want[:, 0] == P.KEPT).sum())
    assert state[0] == kept
    assert state[1] == (P.NO_ABORT if not P.aborted(want) else
                        min(i - i % batch if s == P.NON_FINITE else i for i, s in enumerate(want[:, 0])
                            if s in (P.NON_FINITE, P.EMPTY)))
    got = crops[:kept].cpu().numpy()
    for slot, c in enumerate(P.crops(frames, want)):
        assert np.array_equal(got[slot], PO.resize_linear_u8(c, (96, 96))), slot


def _golden(k):
    frames, has, dets = G[f"c{k}_frames"], G[f"c{k}_has"], G[f"c{k}_dets"]
    return frames, has, dets, [dets[f] if has[f] else None for f in range(len(has))], int(G[f"c{k}_batch"])


@pytest.mark.parametrize("k", range(len(CASES)), ids=CASES)
def test_kernel_matches_oracle_on_golden_cases(k):
    frames, has, dets, top, batch = _golden(k)
    fd = torch.from_numpy(frames).cuda()
    dd = torch.from_numpy(dets).reshape(-1, 1, 5).cuda()
    cd = torch.from_numpy(has.astype(np.int32)).cuda()
    assert P.files(P.preprocess_rows(top, *frames.shape[1:3], batch)) == list(G[f"c{k}_files"])
    for name, calls in _splits(len(has), batch).items():
        rows, state, crops = _run(fd, dd, cd, batch, calls)
        _check(frames, top, batch, rows, state, crops)
    # one frame per call at batch 1 (the oracle at batch 1: a non-finite box loses only its own frame onward)
    rows, state, crops = _run(fd, dd, cd, 1, [1] * len(has))
    _check(frames, top, 1, rows, state, crops)


def test_max_det_rows_past_the_first_are_ignored():
    frames, has, dets, top, batch = _golden(CASES.index("len70"))
    d3 = np.zeros((len(has), 3, 5), dtype=np.float32)
    d3[:, 0] = dets
    d3[:, 1:] = np.nan
    rows, state, crops = _run(torch.from_numpy(frames).cuda(), torch.from_numpy(d3).cuda(),
                              torch.from_numpy(has.astype(np.int32) * 3).cuda(), batch, [len(has)])
    _check(frames, top, batch, rows, state, crops)


@pytest.mark.parametrize("H,W", [(720, 1280), (1080, 1920)])
def test_edge_boxes_at_video_sizes(H, W):
    g = torch.Generator(device="cuda").manual_seed(H)
    F = 9
    frames_d = torch.randint(0, 256, (F, H, W, 3), dtype=torch.uint8, device="cuda", generator=g)
    inf = np.inf
    boxes = [[0, 0, 1e30, 1e30], [100.7, 50.2, 900.9, 700.1], [W - 0.5, 0, 1e30, 10], [-inf, -inf, 5.9, 5.9],
             [W - 40.2, H - 30.9, W + 3e9, H + 7.5], [17.5, 3.0, 60.0, 1e30], None, [3.0, 3.0, 1e30, 2e30],
             [10.0, 10.0, 10.5, 50.0]]   # the last is empty: the video ends there
    has = np.array([b is not None for b in boxes])
    dets = np.array([(b if b is not None else [0, 0, 0, 0]) + [0.9] for b in boxes], dtype=np.float32)
    top = [dets[f] if has[f] else None for f in range(F)]
    frames = frames_d.cpu().numpy()
    for batch, calls in [(4, [4, 4, 1]), (3, [9]), (1, [1] * F)]:
        rows, state, crops = _run(frames_d, torch.from_numpy(dets).reshape(F, 1, 5).cuda(),
                                  torch.from_numpy(has.astype(np.int32)).cuda(), batch, calls)
        _check(frames, top, batch, rows, state, crops)
        assert rows[0].tolist()[2:] == [0, H, 0, W] and rows[1, 0] == 0 and rows[1, 3] - rows[1, 2] > 96
        assert rows[-1, 0] == P.EMPTY


def test_invalid_arguments_and_cap_overflow():
    from wav2lip_b200 import _lib
    ctx = _ctx()
    frames, has, dets, top, batch = _golden(CASES.index("len33"))
    fd, dd = torch.from_numpy(frames).cuda(), torch.from_numpy(dets).reshape(-1, 1, 5).cuda()
    cd = torch.from_numpy(has.astype(np.int32)).cuda()
    F, H, W = frames.shape[:3]
    rows = torch.zeros((F, 6), dtype=torch.int32, device="cuda")
    state = torch.zeros(2, dtype=torch.int32, device="cuda")
    out = torch.zeros((F, 96, 96, 3), dtype=torch.uint8, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    good = dict(frames=_p(fd), B=F, H=H, W=W, dets=_p(dd), counts=_p(cd), max_det=1, frame0=0, batch=32, state=_p(state),
                rows=_p(rows), crops=_p(out), cap=F)
    order = list(good)

    def call(**kw):
        a = dict(good, **kw)
        return ctx.lib.w2l_face_crops_u8(ctx.h, *[a[k] for k in order], st)
    launches = ctx.launch_count()
    for bad in [dict(frames=None), dict(dets=None), dict(counts=None), dict(state=None), dict(rows=None), dict(crops=None),
                dict(B=0), dict(B=-1), dict(H=0), dict(W=-2), dict(max_det=0), dict(batch=0), dict(frame0=5),
                dict(frame0=-32), dict(cap=-1)]:
        assert call(**bad) == _lib.W2L_EINVAL, bad
    pageable = np.zeros((F, 96, 96, 3), dtype=np.uint8)
    assert call(crops=C.c_void_p(pageable.ctypes.data)) == _lib.W2L_EINVAL
    assert ctx.lib.w2l_face_crops_u8(None, *[good[k] for k in order], st) == _lib.W2L_EINVAL
    torch.cuda.synchronize()
    assert ctx.launch_count() == launches and not rows.any() and not out.any()
    # cap overflow: slots >= cap are never written, state[0] reports the kept count
    big = torch.full((F, 96, 96, 3), 77, dtype=torch.uint8, device="cuda")
    rows_h, state_h, crops = _run(fd, dd, cd, batch, [F], cap=5, out=big)
    kept = int((P.preprocess_rows(top, H, W, batch)[:, 0] == 0).sum())
    assert state_h[0] == kept > 5
    assert (crops[5:].cpu().numpy() == 77).all()
    want = P.crops(frames, P.preprocess_rows(top, H, W, batch))
    for slot in range(5):
        assert np.array_equal(crops[slot].cpu().numpy(), PO.resize_linear_u8(want[slot], (96, 96)))
    # face_crops refuses an `out` too small for the kept frames
    from wav2lip_b200 import data as D
    fa = _fa(_net_state(6.0))
    with pytest.raises(ValueError):
        D.face_crops(fa, np.zeros((2, 64, 64, 3), np.uint8), out=torch.zeros((2, 96, 96), dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        D.face_crops(fa, np.zeros((2, 64, 64, 3), np.uint8), batch_size=0)


# ---- 2. end to end with the device detector --------------------------------------------------------------------------------
def _net_state(bg):
    sd = S.make_state_dict(0)
    for i, t in enumerate(TAPS):
        b = sd[f"{t}_mbox_conf.bias"]
        if i == 0:
            b[:3] += bg
        else:
            b[0] += bg
    return sd


def _fa(sd, fa=None):
    """A FaceAlignment on the seeded weights (reloaded into `fa`'s module when given: one context, one set of plans)."""
    from wav2lip_b200.face_detection import FaceAlignment, LandmarksType
    from wav2lip_b200.face_detection.detection.sfd.net_s3fd import s3fd
    if fa is None:
        fa = FaceAlignment(LandmarksType._2D, flip_input=False, device="cuda")
        fa.face_detector.face_detector = s3fd()
    m = fa.face_detector.face_detector
    m.load_state_dict(sd, strict=True)
    fa.face_detector.face_detector = m.cuda().eval()
    return fa


def _video(F, H, W, seed):
    """Noise frames with a run of flat grey ones near the end: the two kinds score differently."""
    v = S.make_images(F, H, W, seed=seed)
    v[F - 6:F - 2] = 100 + seed % 50
    return v


def _oracle_rows(fa, frames, batch):
    top = []
    for s in range(0, len(frames), 32):
        for d in fa.face_detector.detect_from_batch_u8(frames[s:s + 32], max_det=1, reverse_channels=True):
            top.append(d[0] if len(d) else None)
    return P.preprocess_rows(top, frames.shape[1], frames.shape[2], batch)


@pytest.fixture(scope="module", params=[(160, 160), (720, 1280)], ids=["160x160", "720p"])
def setup(request):
    """A detector whose background bias leaves some frames without a face and keeps others, and its videos."""
    H, W = request.param
    F = 40 if H == 160 else 24
    videos = [_video(F, H, W, seed) for seed in (1, 2, 3)]
    fa = None
    for bg in (0.0, 2.0, 4.0, 6.0, 8.0, 10.0, 12.0, 14.0):
        fa = _fa(_net_state(bg), fa)
        rows = [_oracle_rows(fa, v, 32) for v in videos]
        st = np.concatenate([r[:, 0] for r in rows])
        if (st == P.NO_FACE).any() and (st == P.KEPT).sum() >= 20:
            print(f"[{H}x{W}] bg {bg}: statuses {np.bincount(st, minlength=5).tolist()}")
            return fa, videos, rows
    pytest.fail("no background bias gives frames both with and without a face")


def test_face_crops_rows_match_oracle(setup):
    from wav2lip_b200 import data as D
    fa, videos, rows = setup
    assert any((r[:, 0] == P.NO_FACE).any() for r in rows)
    for v, want in zip(videos, rows):
        for src in (v, torch.from_numpy(v).cuda()):
            got, crops = D.face_crops(fa, src)
            assert np.array_equal(got, want)
            assert crops.shape[0] == (want[:, 0] == 0).sum()
            ref = [PO.resize_linear_u8(c, (96, 96)) for c in P.crops(v, want)]
            assert np.array_equal(crops.cpu().numpy(), np.array(ref, dtype=np.uint8).reshape(-1, 96, 96, 3))
    # batch_size only moves the abort point: at 4 the rows equal the oracle's at 4
    got, _ = D.face_crops(fa, videos[0], batch_size=4)
    assert np.array_equal(got, _oracle_rows(fa, videos[0], 4))


def _wav(n, seed):
    return (np.random.default_rng(seed).standard_normal(n) * 0.1).astype(np.float32)


def _sampleable(v):
    ids = sorted(int(n.split(".")[0]) for n in v.img_names)
    run = best = 1
    for a, b in zip(ids, ids[1:]):
        run = run + 1 if b == a + 1 else 1
        best = max(best, run)
    return len(ids) > 15 and best >= 12 and v.mel_len >= 60


def test_from_videos_equals_from_arrays(setup):
    from wav2lip_b200 import audio
    from wav2lip_b200 import data as D
    fa, videos, rows = setup
    srs = [16000, 48000, 16000]
    wavs = [_wav(int(len(v) / 25 * sr) + 123, i) for i, (v, sr) in enumerate(zip(videos, srs))]
    wavs[2] = None                                              # the audio failed
    vids = [{"path": f"v{i}", "frames": v if i else torch.from_numpy(v).cuda(), "wav": w, "sr": sr}
            for i, (v, w, sr) in enumerate(zip(videos, wavs, srs))]
    arrays = []
    for i, (v, r, w, sr) in enumerate(zip(videos, rows, wavs, srs)):
        keep = np.flatnonzero(r[:, 0] == 0)
        wav16 = None if w is None else (w if sr == 16000 else audio.resample(w, sr, 16000))
        arrays.append({"path": f"v{i}", "img_names": [f"{j}.jpg" for j in keep], "wav": wav16,
                       "crops": [v[j][r[j, 2]:r[j, 3], r[j, 4]:r[j, 5]] for j in keep]})
    for storage in ("device", "pinned"):
        a = D.TrainDataCache.from_videos(iter(vids), fa, storage=storage)
        b = D.TrainDataCache.from_arrays(arrays, storage=storage)
        assert a.frames.is_cuda == (storage == "device") and (storage == "device" or a.frames.is_pinned())
        assert a.frames.shape == b.frames.shape and torch.equal(a.frames.cpu(), b.frames.cpu())
        for x, y in zip(a.videos, b.videos):
            assert (x.path, x.img_names, x.slots, x.mel_off, x.mel_len) == (y.path, y.img_names, y.slots, y.mel_off, y.mel_len)
        assert a.videos[2].mel_len == -1
        assert torch.equal(a.mels, b.mels)
        m48 = audio.melspectrogram(audio.resample(torch.from_numpy(wavs[1]).cuda(), 48000, 16000)).t()
        assert torch.equal(a.mels[a.videos[1].mel_off:a.videos[1].mel_off + a.videos[1].mel_len], m48)
        if all(_sampleable(v) for v in a.videos[:2]):   # else the samplers would redraw forever
            for cls in (D.Wav2LipBatches, D.SyncNetBatches):
                ba = cls(a, 4, rng=random.Random(5)).next_batch()
                bb = cls(b, 4, rng=random.Random(5)).next_batch()
                assert all(torch.equal(x, y) for x, y in zip(ba, bb))
