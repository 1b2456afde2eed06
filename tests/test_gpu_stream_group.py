"""Stream groups on the GPU: `stream.LipSyncServer` against the offline composition of inference.py (`_offline`, as in
test_gpu_stream.py, with the frame size of each video) and against a lone `LipSyncSession` fed the same pieces, bit for
bit and frame for frame, for mixed sessions and tick patterns; NaN isolation, new weights, graph on/off, pinned bucket
plans, bounded memory, per-tick call counts and argument checks."""
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


@pytest.fixture(scope="module")
def gen():
    from wav2lip_b200.models import Wav2Lip
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
    return g.cuda().eval()


def _model(seed=0):
    from wav2lip_b200.models import Wav2Lip
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", seed, init="default"), strict=True)
    return g.cuda().eval()


def _video(F, H, W, seed):
    rng = np.random.default_rng(seed)
    frames = torch.from_numpy(rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)).cuda()
    return frames, random_rects(rng, F, H, W)


def _offline(g, frames, wav, fps, rects=None, box=None, nosmooth=False, pads=(0, 10, 0, 0), batch=128):
    from wav2lip_b200 import audio
    from wav2lip_b200.face_detection import face_boxes
    H, W = frames.shape[1:3]
    mel = audio.melspectrogram(wav)
    chunks = torch.from_numpy(audio.mel_chunks(mel, fps)).cuda()
    n = chunks.shape[0]
    n_total = min(n, frames.shape[0])
    if box is not None:
        bx = np.asarray([box] * n_total, dtype=np.int64)
    else:
        bx = face_boxes([tuple(int(v) for v in r) for r in rects[:n_total]], H, W, pads, nosmooth)
    rows = np.asarray([(i % n_total,) + tuple(bx[i % n_total]) for i in range(n)], dtype=np.int32)
    with torch.no_grad():
        return torch.cat([g.infer_frames(chunks[k:k + batch], frames, rows[k:k + batch]) for k in range(0, n, batch)])


def _lone(g, frames, fps, pieces, batch, **kw):
    from wav2lip_b200.stream import LipSyncSession
    s = LipSyncSession(g, frames, fps, batch=batch, **kw)
    outs = [s.push(p)[1] for p in pieces] + [s.finish()[1]]
    s.close()
    return torch.cat(outs)


def _pieces(rng, wav, kind):
    """wav cut into 640-sample pieces or pieces of random length"""
    n = wav.shape[0]
    if kind == "640":
        sizes = [640] * (n // 640) + ([n % 640] if n % 640 else [])
    else:
        sizes, left = [], n
        while left:
            k = int(min(left, rng.integers(1, 5000)))
            sizes.append(k)
            left -= k
    at = np.cumsum([0] + sizes)
    return [wav[at[i]:at[i + 1]] for i in range(len(sizes))]


class _Run:
    """Drives sessions of one server: each tick gives a random subset of the sessions their next piece (the others
    idle), finishes a session with its last piece or in a later tick, and checks that output indices continue."""

    def __init__(self, srv, rng):
        self.srv, self.rng = srv, rng
        self.pieces, self.outs, self.next, self.done, self.expect = {}, {}, {}, {}, {}

    def add(self, sid, pieces):
        self.pieces[sid], self.outs[sid], self.next[sid], self.done[sid], self.expect[sid] = pieces, [], 0, False, 0

    def tick(self):
        live = [s for s in self.pieces if not self.done[s]]
        if not live:
            return False
        chosen = [s for s in live if self.rng.random() < 0.7] or live[:1]
        pieces, fin = {}, []
        for s in chosen:
            k = self.next[s]
            if k < len(self.pieces[s]):
                pieces[s] = self.pieces[s][k]
                self.next[s] = k + 1
                if self.next[s] == len(self.pieces[s]) and self.rng.random() < 0.5:
                    fin.append(s)
            else:
                fin.append(s)
        res = self.srv.tick(pieces, finish=fin)
        assert set(res) == set(pieces) | set(fin)
        for s, (first, fr) in res.items():
            assert first == self.expect[s]
            self.expect[s] += fr.shape[0]
            self.outs[s].append(fr)
        for s in fin:
            self.done[s] = True
        return True

    def result(self, sid):
        return torch.cat(self.outs[sid])


CASES = [  # (F, seconds of audio, fps, nosmooth, box, H, W)
    (12, 0.30, 25.0, False, None, 64, 96),        # audio shorter than the video
    (12, 0.60, 25.0, False, None, 96, 72),        # as many chunks as frames
    (12, 1.30, 25.0, False, None, 57, 91),        # longer; frames not 16-byte aligned
    (1, 0.70, 25.0, False, None, 88, 120),        # a still image
    (12, 0.90, 29.97002997, True, None, 72, 88),  # nosmooth
    (12, 0.90, 29.97002997, False, (5, 60, 7, 80), 72, 88),   # a fixed box
]


def _case(c):
    F, sec, fps, nosmooth, box, H, W = CASES[c]
    frames, rects = _video(F, H, W, seed=c)
    n = int(sec * 16000) + 37 * c
    wav = M.make_wav(n, seed=c, kind="mix")
    return frames, wav, fps, dict(rects=None if box else rects, box=box, nosmooth=nosmooth)


@pytest.mark.parametrize("max_batch", [1, 4, 16])
@pytest.mark.parametrize("kind", ["640", "random"])
def test_group_matches_offline_and_lone_session(gen, max_batch, kind):
    from wav2lip_b200.stream import LipSyncServer
    rng = np.random.default_rng(max_batch * 7 + len(kind))
    srv = LipSyncServer(gen, max_batch=max_batch)
    run, cases = _Run(srv, rng), {}
    for c in range(len(CASES)):
        frames, wav, fps, kw = _case(c)
        sid = srv.open(frames, fps, **kw)
        cases[sid] = (c, frames, wav, fps, kw, _pieces(rng, wav, kind))
        run.add(sid, cases[sid][5])
    while run.tick():
        pass
    for sid, (c, frames, wav, fps, kw, pieces) in cases.items():
        got = run.result(sid)
        ref = _offline(gen, frames, wav, fps, **kw)
        assert got.shape == ref.shape, c
        assert torch.equal(got, ref), c
        assert torch.equal(got, _lone(gen, frames, fps, pieces, 4, **kw)), c
    srv.close()


def test_sessions_opened_and_closed_mid_run(gen):
    from wav2lip_b200.stream import LipSyncServer
    rng = np.random.default_rng(3)
    srv = LipSyncServer(gen, max_batch=8)
    run = _Run(srv, rng)
    fa, wa, fpa, kwa = _case(2)
    fb, wb, fpb, kwb = _case(4)
    a = srv.open(fa, fpa, **kwa)
    b = srv.open(fb, fpb, **kwb)
    run.add(a, _pieces(rng, wa, "640"))
    run.add(b, _pieces(rng, wb, "random"))
    for _ in range(5):
        run.tick()
    srv.close(b)                              # closed unfinished
    del run.pieces[b]
    fc, wc, fpc, kwc = _case(5)
    c = srv.open(fc, fpc, **kwc)              # may reuse b's slot
    run.add(c, _pieces(rng, wc, "640"))
    while run.tick():
        pass
    assert torch.equal(run.result(a), _offline(gen, fa, wa, fpa, **kwa))
    assert torch.equal(run.result(c), _offline(gen, fc, wc, fpc, **kwc))
    with pytest.raises(Exception):
        srv.tick({b: wb[:640]})
    srv.close()


def test_nan_fails_one_session_only(gen):
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(gen, max_batch=4)
    vids = [_video(60, 72, 88, seed=20 + k) for k in range(3)]
    wavs = [M.make_wav(32000, seed=20 + k, kind="mix") for k in range(3)]
    bad = wavs[1].copy()
    bad[20000] = np.nan
    feed = [wavs[0], bad, wavs[2]]
    ids = [srv.open(f, 25.0, rects=r) for f, r in vids]
    outs = [[], [], []]
    failed_at = None
    for i in range(50):
        res = srv.tick({ids[k]: feed[k][i * 640:(i + 1) * 640] for k in range(3) if failed_at is None or k != 1})
        for k in range(3):
            if ids[k] not in res:
                continue
            v = res[ids[k]]
            if isinstance(v, ValueError):
                assert k == 1 and failed_at is None
                assert str(v).startswith("Mel contains nan! Using a TTS voice?")
                failed_at = i
                continue
            outs[k].append(v[1])
    assert failed_at == 31      # as LipSyncSession: the piece that makes frame 99 final (test_gpu_stream.py)
    with pytest.raises(ValueError, match="Mel contains nan!"):
        srv.tick({ids[1]: wavs[1][:640], ids[0]: wavs[0][:0]})
    res = srv.tick({}, finish=[ids[0], ids[2]])
    for k in (0, 2):
        outs[k].append(res[ids[k]][1])
        assert torch.equal(torch.cat(outs[k]), _offline(gen, vids[k][0], wavs[k][:32000], 25.0, rects=vids[k][1]))
    got = torch.cat(outs[1])
    clean = _offline(gen, vids[1][0], wavs[1], 25.0, rects=vids[1][1])
    assert torch.equal(got, clean[:got.shape[0]])
    srv.close()


def test_new_weights_between_ticks():
    from wav2lip_b200.stream import LipSyncServer
    g = _model(0)
    srv = LipSyncServer(g, max_batch=4)
    frames, rects = _video(40, 72, 88, seed=7)
    wav = M.make_wav(16000, seed=7, kind="mix")
    a = srv.open(frames, 25.0, rects=rects)
    outs = [srv.tick({a: wav[i * 640:(i + 1) * 640]})[a][1] for i in range(12)]
    n_old = sum(o.shape[0] for o in outs)
    ref_old = _offline(g, frames, wav, 25.0, rects=rects)
    g.load_state_dict(O.make_state_dict("generator", 1, init="default"), strict=True)
    outs += [srv.tick({a: wav[i * 640:(i + 1) * 640]})[a][1] for i in range(12, 25)]
    outs.append(srv.tick({}, finish=[a])[a][1])
    srv.close()
    got = torch.cat(outs)
    ref_new = _offline(g, frames, wav, 25.0, rects=rects)
    assert n_old > 0 and got.shape == ref_new.shape
    assert torch.equal(got[:n_old], ref_old[:n_old])
    assert torch.equal(got[n_old:], ref_new[n_old:])


def test_graph_on_and_off_identical(monkeypatch):
    from wav2lip_b200.stream import LipSyncServer
    results = []
    for off in ("0", "1"):
        monkeypatch.setenv("W2L_DISABLE_STREAMGRAPH", off)
        g = _model(0)
        srv = LipSyncServer(g, max_batch=8)
        run = _Run(srv, np.random.default_rng(11))
        for c in (0, 2, 5):
            frames, wav, fps, kw = _case(c)
            run.add(srv.open(frames, fps, **kw), _pieces(np.random.default_rng(c), wav, "random"))
        while run.tick():
            pass
        results.append([run.result(s) for s in sorted(run.pieces)])
        srv.close()
    for x, y in zip(*results):
        assert torch.equal(x, y)


def test_pinned_bucket_plans_survive_lru_eviction(gen):
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(gen, max_batch=4)
    frames, rects = _video(12, 72, 88, seed=12)
    wav = M.make_wav(24000, seed=12, kind="mix")
    a = srv.open(frames, 25.0, rects=rects)
    outs = [srv.tick({a: wav[i * 640:(i + 1) * 640]})[a][1] for i in range(14)]    # graphs captured by now
    chunks = torch.rand(11, 1, 80, 16, device="cuda")
    rows = np.asarray([(j % 12, 5, 60, 7, 80) for j in range(11)], dtype=np.int32)
    with torch.no_grad():
        for N in (3, 5, 6, 7, 9, 10, 11):            # other plans: more than the LRU keeps
            gen.infer_frames(chunks[:N], frames, rows[:N])
    outs += [srv.tick({a: wav[i * 640:(i + 1) * 640]})[a][1] for i in range(14, 38)]
    outs.append(srv.tick({}, finish=[a])[a][1])
    srv.close()
    assert torch.equal(torch.cat(outs), _offline(gen, frames, wav, 25.0, rects=rects))


def test_long_run_small_ring_constant_memory(gen):
    """Two sessions, 40 s each through 2^11-sample audio rings: device memory after 1 s equals that after 40 s."""
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(gen, max_batch=4, audio_ring_log2=11)
    vids = [_video(30, 72, 88, seed=30 + k) for k in range(2)]
    n = 16000 * 40 + 123
    wavs = [(0.1 * np.sin(np.arange(n) * (0.011 + 0.002 * k))
             + 0.01 * np.random.default_rng(k).standard_normal(n)).astype(np.float32) for k in range(2)]
    ids = [srv.open(vids[0][0], 25.0, rects=vids[0][1]), srv.open(vids[1][0], 29.97002997, box=(5, 60, 7, 80))]
    outs, mem_1s = [[], []], None
    ctx = gen._w2l_ctx
    for i, at in enumerate(range(0, n, 640)):
        res = srv.tick({ids[k]: wavs[k][at:at + 640] for k in range(2)})
        for k in range(2):
            outs[k].append(res[ids[k]][1])
        if at >= 16000 and mem_1s is None:
            torch.cuda.synchronize()
            mem_1s = ctx.device_bytes()
    torch.cuda.synchronize()
    assert ctx.device_bytes() == mem_1s
    res = srv.tick({}, finish=ids)
    for k in range(2):
        outs[k].append(res[ids[k]][1])
    assert torch.equal(torch.cat(outs[0]), _offline(gen, vids[0][0], wavs[0], 25.0, rects=vids[0][1]))
    assert torch.equal(torch.cat(outs[1]), _offline(gen, vids[1][0], wavs[1], 29.97002997, box=(5, 60, 7, 80)))
    srv.close()


def test_calls_per_tick_do_not_grow_with_sessions(gen):
    """A tick of 2 sessions and a tick of 64 that each fit one step make the same CUDA calls and host waits."""
    from wav2lip_b200.stream import LipSyncServer
    frames, _ = _video(4, 72, 88, seed=40)
    wav = M.make_wav(16000 * 2, seed=40, kind="mix")
    deltas = []
    for count in (2, 64):
        srv = LipSyncServer(gen, max_batch=128)
        ids = [srv.open(frames, 25.0, box=(5, 60, 7, 80)) for _ in range(count)]
        for i in range(30):                              # every bucket these ticks use is captured
            srv.tick({s: wav[i * 640:(i + 1) * 640] for s in ids})
        c0, l0 = srv.counters(), gen._w2l_ctx.launch_count()
        res = srv.tick({s: wav[30 * 640:31 * 640] for s in ids})
        c1, l1 = srv.counters(), gen._w2l_ctx.launch_count()
        assert all(res[s][1].shape[0] >= 1 for s in ids)
        assert c1[2] - c0[2] == 1                        # one step
        deltas.append((c1[0] - c0[0], c1[1] - c0[1], l1 - l0))
        srv.close()
    assert deltas[0] == deltas[1]
    assert deltas[0][1] == 2                             # the NaN read-back and the table staging slot


def test_bad_arguments_rejected_before_launch(gen):
    from wav2lip_b200 import _lib
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(gen, max_batch=4)
    frames, rects = _video(6, 72, 88, seed=11)
    wav = M.make_wav(16000, seed=11, kind="mix")
    a = srv.open(frames, 25.0, rects=rects)
    outs = [srv.tick({a: wav[:640]})[a][1]]
    launches, counters = gen._w2l_ctx.launch_count(), srv.counters()
    with pytest.raises(ValueError):
        srv.open(frames, 25.0, rects=[tuple(r) for r in rects[:5]] + [None])
    with pytest.raises(_lib.W2LError):
        srv.open(frames, 25.0, box=(5, 80, 7, 80))       # outside the 72-row frame
    with pytest.raises(_lib.W2LError):
        srv.open(frames.cpu(), 25.0, rects=rects)
    b = srv.open(frames, 25.0, box=(5, 60, 7, 80))
    srv.close(b)
    with pytest.raises(_lib.W2LError):
        srv.tick({a: wav[640:1280], b: wav[:640]})       # a closed session
    with pytest.raises(_lib.W2LError):
        srv.tick({a: wav[640:1280], 12345: wav[:640]})   # never opened
    assert gen._w2l_ctx.launch_count() == launches and srv.counters() == counters
    outs += [srv.tick({a: wav[i * 640:(i + 1) * 640]})[a][1] for i in range(1, 25)]
    outs.append(srv.tick({}, finish=[a])[a][1])
    assert torch.equal(torch.cat(outs), _offline(gen, frames, wav[:16000], 25.0, rects=rects))
    srv.close()
