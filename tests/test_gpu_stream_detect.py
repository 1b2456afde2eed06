"""Face detection inside the stream server (`LipSyncServer(..., detector=fa)`, `open(frames, fps)` without rects or box,
include/w2l.h `w2l_stream_group_open_detect`, DESIGN.md section 3.10) on the GPU.

Each detected session is compared, bit for bit and frame for frame, with the composition inference.py makes:
`fa.get_detections_for_batch_u8(frames[:n_total])` in batches of 16 -> `face_boxes` -> `infer_frames` (`_offline` of
test_gpu_stream_group.py), and with a session of the same server opened with those rects.  The detector has random S3FD
weights (`make_state_dict`, loc heads scaled down so that boxes stay inside the frame); the tests assert that the frames
they need have faces and that the rects differ between frames.  Also: S3FD batch invariance at 720p (the server detects
in batches of 1, 4 and 16, the composition in 16s), frames without a face before and past the end of the utterance, a
non-finite top box, calls per tick, graph on / off, constant device memory, new detector weights between ticks, and the
precision check."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import mel_oracle as M
from oracle import s3fd_oracle as S

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_s3fd_detect import _net, _raise_bg, _same_bits, _tie_state  # noqa: E402
from test_gpu_stream_group import CASES, _offline, _pieces, _Run  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gen():
    from oracle import w2l_oracle as O
    from wav2lip_b200.models import Wav2Lip
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
    return g.cuda().eval()


def _near_anchors(sd):
    """Random S3FD weights with the loc heads scaled by 1e-3: every box stays within a few pixels of its anchor, so the
    padded boxes are non-empty and inside the frame, as inference.py needs them to be."""
    for k in sd:
        if "_mbox_loc." in k:
            sd[k] *= 1e-3
    return sd


def _fa(sd):
    from wav2lip_b200.face_detection import FaceAlignment, LandmarksType
    fa = FaceAlignment(LandmarksType._2D, flip_input=False, device="cuda")
    fa.face_detector.face_detector = _net(sd)
    return fa


@pytest.fixture(scope="module")
def fa():
    return _fa(_near_anchors(S.make_state_dict(0)))


def _detect_all(fa, frames):
    out = []
    for k in range(0, frames.shape[0], 16):    # inference.py's --face_det_batch_size default
        out += fa.get_detections_for_batch_u8(frames[k:k + 16])
    return out


def _n_total(wav, fps, F):
    from wav2lip_b200 import audio
    return min(audio.mel_chunks(audio.melspectrogram(wav), fps).shape[0], F)


def _composition(gen, fa, frames, wav, fps, nosmooth, distinct=True):
    """inference.py's order: detect frames[:n_total], then boxes, then the generator -> (frames, rects)."""
    rects = _detect_all(fa, frames[:_n_total(wav, fps, frames.shape[0])])
    assert all(r is not None for r in rects)
    assert not distinct or len(rects) == 1 or len(set(rects)) > 1
    return _offline(gen, frames, wav, fps, rects=rects, nosmooth=nosmooth), rects


def _case(c):
    F, sec, fps, nosmooth, box, H, W = CASES[c]
    rng = np.random.default_rng(100 + c)
    frames = torch.from_numpy(rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)).cuda()
    wav = M.make_wav(int(sec * 16000) + 37 * c, seed=c, kind="mix")
    return frames, wav, fps, nosmooth, box


@pytest.mark.parametrize("max_batch", [1, 16])
@pytest.mark.parametrize("kind", ["640", "random"])
def test_detected_sessions_match_composition(gen, fa, max_batch, kind):
    from wav2lip_b200.stream import LipSyncServer
    rng = np.random.default_rng(max_batch * 5 + len(kind))
    srv = LipSyncServer(gen, max_batch=max_batch, detector=fa)
    run, cases = _Run(srv, rng), {}
    for c in range(len(CASES)):
        frames, wav, fps, nosmooth, box = _case(c)
        pieces = _pieces(rng, wav, kind)
        if box is not None:            # a fixed-box session beside the detected ones
            sid = srv.open(frames, fps, box=box)
            cases[sid] = (frames, wav, fps, None, None, box)
            run.add(sid, pieces)
            continue
        ref, rects = _composition(gen, fa, frames, wav, fps, nosmooth)
        all_rects = _detect_all(fa, frames)
        all_rects = [r if r is not None else rects[0] for r in all_rects]
        a = srv.open(frames, fps, nosmooth=nosmooth)
        b = srv.open(frames, fps, rects=all_rects, nosmooth=nosmooth)
        cases[a] = (frames, wav, fps, nosmooth, ref, None)
        cases[b] = (frames, wav, fps, nosmooth, ref, None)
        run.add(a, pieces)
        run.add(b, pieces)
    while run.tick():
        pass
    for sid, (frames, wav, fps, nosmooth, ref, box) in cases.items():
        got = run.result(sid)
        if box is not None:
            ref = _offline(gen, frames, wav, fps, box=box)
        assert got.shape == ref.shape, sid
        assert torch.equal(got, ref), sid
    srv.close()


def test_s3fd_batch_invariance_at_720p(fa):
    net = fa.face_detector.face_detector
    frames = torch.from_numpy(S.make_images(16, 720, 1280, seed=21)).cuda()
    with torch.no_grad():
        d16, c16, m16 = net.detect_u8(frames, 1, reverse_channels=True, return_maps=True)
        for b in (0, 9, 15):
            d1, c1, m1 = net.detect_u8(frames[b:b + 1], 1, reverse_channels=True, return_maps=True)
            for x, y in zip(m1, m16):
                assert torch.equal(x[0].view(torch.int32), y[b].view(torch.int32)), b
            assert int(c1[0]) == int(c16[b]) and _same_bits(d1[0].cpu().numpy(), d16[b].cpu().numpy()), b


def _feed(srv, sessions, ticks):
    """sessions: {id: wav}; 640-sample pieces, each session finished with its last piece -> ({id: [frames...]},
    {id: (tick, error)})."""
    outs, errs = {s: [] for s in sessions}, {}
    for t in range(ticks):
        live = {s: w for s, w in sessions.items() if s not in errs and t * 640 < w.shape[0]}
        if not live:
            break
        fin = [s for s, w in live.items() if (t + 1) * 640 >= w.shape[0]]
        res = srv.tick({s: w[t * 640:(t + 1) * 640] for s, w in live.items()}, finish=fin)
        for s, v in res.items():
            if isinstance(v, ValueError):
                errs[s] = (t, v)
            else:
                outs[s].append(v[1])
    return {s: torch.cat(v) if v else None for s, v in outs.items()}, errs


def test_frames_without_a_face(gen):
    from wav2lip_b200.stream import LipSyncServer, detect_need
    rng = np.random.default_rng(31)
    pool = torch.from_numpy(rng.integers(0, 256, (48, 72, 88, 3), dtype=np.uint8)).cuda()
    base = _near_anchors(S.make_state_dict(0))
    fa = _fa(base)
    lo, hi = 0.0, 512.0
    for _ in range(40):   # bisect the background bias until the detector itself finds both kinds in the pool
        bg = (lo + hi) / 2
        fa.face_detector.face_detector.load_state_dict(_raise_bg({k: v.clone() for k, v in base.items()}, bg))
        kinds = _detect_all(fa, pool)
        face = [i for i, r in enumerate(kinds) if r is not None]
        none = [i for i, r in enumerate(kinds) if r is None]
        if len(face) >= 13 and len(none) >= 2:
            break
        lo, hi = (lo, bg) if len(face) < 13 else (bg, hi)
    assert len(face) >= 13 and len(none) >= 2, (bg, len(face), len(none))
    F = 12
    vid_a = pool[face[:F]].clone()
    vid_a[5] = pool[none[0]]                     # past n_total = 5 of a 0.3 s utterance, but inside the prefetch
    vid_b = pool[face[:F]].clone()
    vid_b[7] = pool[none[1]]                     # inside the utterance
    vid_c = pool[face[1:F + 1]].clone()
    wav_a = M.make_wav(4800, seed=1, kind="mix")
    wav_b = M.make_wav(20800, seed=2, kind="mix")
    wav_c = M.make_wav(20800, seed=3, kind="mix")
    assert _n_total(wav_a, 25.0, F) == 5
    assert detect_need(4800 + 3200, F, 72, 88, 25.0) > 5
    srv = LipSyncServer(gen, max_batch=4, detector=fa)
    a, b, c = srv.open(vid_a, 25.0), srv.open(vid_b, 25.0), srv.open(vid_c, 25.0)
    outs, errs = _feed(srv, {a: wav_a, b: wav_b, c: wav_c}, 40)
    assert set(errs) == {b}
    t_fail, err = errs[b]
    assert str(err) == "Face not detected in frame 7! Ensure the video contains a face in all the frames."
    first_tick = next(t for t in range(40) if detect_need(640 * (t + 1), F, 72, 88, 25.0) > 7)
    assert t_fail == first_tick
    with pytest.raises(ValueError, match="frame 7"):
        srv.tick({b: wav_b[:640]})
    # (the raised background leaves the largest anchors on top: the rects of these videos may all be equal)
    assert torch.equal(outs[a], _composition(gen, fa, vid_a, wav_a, 25.0, False, distinct=False)[0])
    assert torch.equal(outs[c], _composition(gen, fa, vid_c, wav_c, 25.0, False, distinct=False)[0])
    rects_b = _detect_all(fa, vid_b)
    rects_b[7] = rects_b[0]
    ref_b = _offline(gen, vid_b, wav_b, 25.0, rects=rects_b)
    assert outs[b] is not None and 0 < outs[b].shape[0] < ref_b.shape[0]
    assert torch.equal(outs[b], ref_b[:outs[b].shape[0]])
    srv.close()


def test_non_finite_top_box_fails_the_session(gen):
    from wav2lip_b200.stream import LipSyncServer, detect_need
    fa = _fa(_tie_state((0, 2), (0.0, 0.0, 500.0, 500.0)))
    frames = torch.from_numpy(S.make_images(6, 128, 128, seed=7)).cuda()
    d, cnt, _ = fa.face_detector.face_detector.detect_u8(frames[:1], 1, reverse_channels=True)
    assert int(cnt[0]) == 1 and not torch.isfinite(d[0, 0, :4]).all()
    srv = LipSyncServer(gen, max_batch=4, detector=fa)
    s = srv.open(frames, 25.0)
    wav = M.make_wav(16000, seed=5, kind="mix")
    _, errs = _feed(srv, {s: wav}, 30)
    t_fail, err = errs[s]
    assert str(err) == "Face detector returned a non-finite box in frame 0"
    assert t_fail == next(t for t in range(30) if detect_need(640 * (t + 1), 6, 128, 128, 25.0) > 0)
    srv.close()


def test_calls_per_tick_do_not_grow_with_sessions(gen, fa):
    """9 and 16 detected sessions of one frame size, each needing one more frame in the measured tick: one detection
    launch and one step either way, so the same CUDA calls, launches and host waits."""
    from wav2lip_b200.stream import LipSyncServer, detect_need
    frames = torch.from_numpy(np.random.default_rng(41).integers(0, 256, (60, 72, 88, 3), dtype=np.uint8)).cuda()
    wav = M.make_wav(16000 * 3, seed=41, kind="mix")
    ahead = [detect_need(640 * (t + 1) + 3200, 60, 72, 88, 25.0) for t in range(60)]
    t = next(t for t in range(30, 60) if ahead[t] - ahead[t - 1] == 1)
    deltas = []
    for count in (9, 16):
        srv = LipSyncServer(gen, max_batch=128, detector=fa)
        ids = [srv.open(frames, 25.0) for _ in range(count)]
        for i in range(t):
            srv.tick({s: wav[i * 640:(i + 1) * 640] for s in ids})
        c0, l0 = srv.counters(), gen._w2l_ctx.launch_count()
        res = srv.tick({s: wav[t * 640:(t + 1) * 640] for s in ids})
        c1, l1 = srv.counters(), gen._w2l_ctx.launch_count()
        assert all(not isinstance(res[s], Exception) for s in ids)
        assert c1[2] - c0[2] <= 1
        deltas.append((c1[0] - c0[0], c1[1] - c0[1], c1[2] - c0[2], l1 - l0))
        srv.close()
    assert deltas[0] == deltas[1]
    assert deltas[0][1] == 1 + deltas[0][2]   # the NaN read-back, which also reads the rects back, and a table slot


def test_graph_on_and_off_identical(monkeypatch):
    from oracle import w2l_oracle as O
    from wav2lip_b200.models import Wav2Lip
    from wav2lip_b200.stream import LipSyncServer
    results = []
    for off in ("0", "1"):
        monkeypatch.setenv("W2L_DISABLE_STREAMGRAPH", off)
        g = Wav2Lip()
        g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
        g = g.cuda().eval()
        srv = LipSyncServer(g, max_batch=8, detector=_fa(_near_anchors(S.make_state_dict(0))))
        run = _Run(srv, np.random.default_rng(11))
        for c in (0, 2, 4):
            frames, wav, fps, nosmooth, _ = _case(c)
            run.add(srv.open(frames, fps, nosmooth=nosmooth), _pieces(np.random.default_rng(c), wav, "random"))
        while run.tick():
            pass
        results.append([run.result(s) for s in sorted(run.pieces)])
        srv.close()
    for x, y in zip(*results):
        assert torch.equal(x, y)


def test_long_run_constant_memory(gen, fa):
    """Two detected sessions, 40 s each through 2^11-sample rings: device memory after 2 s (every frame detected, the
    plans built) equals that after 40 s."""
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(gen, max_batch=4, audio_ring_log2=11, detector=fa)
    rng = np.random.default_rng(51)
    vids = [torch.from_numpy(rng.integers(0, 256, (30, 72, 88, 3), dtype=np.uint8)).cuda() for _ in range(2)]
    n = 16000 * 40 + 123
    wavs = [(0.1 * np.sin(np.arange(n) * (0.011 + 0.002 * k))
             + 0.01 * np.random.default_rng(k).standard_normal(n)).astype(np.float32) for k in range(2)]
    fps = (25.0, 29.97002997)
    ids = [srv.open(vids[k], fps[k]) for k in range(2)]
    outs, mem_2s = [[], []], None
    ctx = gen._w2l_ctx
    for at in range(0, n, 640):
        res = srv.tick({ids[k]: wavs[k][at:at + 640] for k in range(2)})
        for k in range(2):
            outs[k].append(res[ids[k]][1])
        if at >= 32000 and mem_2s is None:
            torch.cuda.synchronize()
            mem_2s = ctx.device_bytes()
    torch.cuda.synchronize()
    assert ctx.device_bytes() == mem_2s
    res = srv.tick({}, finish=ids)
    for k in range(2):
        outs[k].append(res[ids[k]][1])
        ref, _ = _composition(gen, fa, vids[k], wavs[k], fps[k], False)
        assert torch.equal(torch.cat(outs[k]), ref), k
    srv.close()


def test_new_detector_weights_apply_to_frames_detected_afterwards(gen):
    from wav2lip_b200.stream import LipSyncServer, detect_need
    fa = _fa(_near_anchors(S.make_state_dict(0)))
    frames = torch.from_numpy(np.random.default_rng(61).integers(0, 256, (40, 72, 88, 3), dtype=np.uint8)).cuda()
    wav = M.make_wav(16000 * 2, seed=61, kind="mix")
    rects_old = _detect_all(fa, frames)
    srv = LipSyncServer(gen, max_batch=4, detector=fa)
    s = srv.open(frames, 25.0)
    outs = [srv.tick({s: wav[i * 640:(i + 1) * 640]})[s][1] for i in range(10)]
    launched = max(detect_need(6400, 40, 72, 88, 25.0), detect_need(6400 + 3200, 40, 72, 88, 25.0))
    fa.face_detector.face_detector.load_state_dict(_near_anchors(S.make_state_dict(1)), strict=True)
    rects_new = _detect_all(fa, frames)
    assert rects_new[launched:] != rects_old[launched:]
    for i in range(10, 50):
        if i * 640 >= wav.shape[0]:
            break
        outs.append(srv.tick({s: wav[i * 640:(i + 1) * 640]})[s][1])
    outs.append(srv.tick({}, finish=[s])[s][1])
    srv.close()
    rects = rects_old[:launched] + rects_new[launched:]
    assert all(r is not None for r in rects[:_n_total(wav, 25.0, 40)])
    assert torch.equal(torch.cat(outs), _offline(gen, frames, wav, 25.0, rects=rects))


def test_precision_mismatch_and_missing_detector_raise(gen):
    from wav2lip_b200 import _lib
    from wav2lip_b200.stream import LipSyncServer
    fa = _fa(S.make_state_dict(0))
    fa.face_detector.face_detector.precision = _lib.PREC_BF16
    with pytest.raises(ValueError, match="precision"):
        LipSyncServer(gen, detector=fa)
    srv = LipSyncServer(gen, max_batch=4)
    frames = torch.zeros((4, 72, 88, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError, match="rects of every frame or one fixed box"):
        srv.open(frames, 25.0)
    srv.close()
