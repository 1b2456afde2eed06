"""The frame side of lip-sync at video sizes (720p, 1080p, 4K and an odd 1079 x 1917), on the GPU: the two cv2.resize
calls and the paste of inference.py (:126, :269-271), in the offline kernels (`Wav2Lip.crop_resize`, `paste`,
`infer_frames`: resize.cuh) and in the stream steps' per-row forms (`LipSyncServer`, `LipSyncSession`: stream.cuh).

These kernels are integer arithmetic, so every check is bit for bit: against the cv2-pinned oracle
(oracle/pipeline_oracle.py, pinned at these sizes by tests/golden/resize_video.json) and, for the streams, against the
offline composition (`_offline` of test_gpu_stream_group.py).  The sizes reach what toy frames do not: crops that
downscale 2 to 20x and pastes that upscale 96 px to 900 px and to whole frames, boxes on every edge and corner, 1 px and
8 px boxes, frames whose byte count is not a multiple of 16 (the stream paste's last, partial 16-byte piece, in each of
its three pixel phases), frames that take several passes of the stream paste's grid-stride loop, one paste launch over
rows of different frame sizes with padding rows, and videos that start at an odd byte address."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import mel_oracle as M
from oracle import pipeline_oracle as P
from oracle import w2l_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from stream_offline import offline_rows  # noqa: E402
from test_gpu_stream_group import _offline, _pieces, _Run  # noqa: E402
from test_pipeline_rows import _gold_image, _sha256, _video_gold  # noqa: E402

pytestmark = pytest.mark.gpu

# 1079 x 1917 x 3 = 6205329 bytes = 16 * 387833 + 1: the stream paste's last piece holds one byte, the last channel of
# the bottom-right pixel
SIZES = [(720, 1280), (1080, 1920), (2160, 3840), (1079, 1917)]


@pytest.fixture(scope="module")
def gen():
    from wav2lip_b200.models import Wav2Lip
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
    return g.cuda().eval()


def _frames(F, H, W, seed, offset=0):
    """(host, CUDA) copies of F seeded (H, W, 3) uint8 frames; offset > 0: the CUDA frames are a contiguous view that
    starts `offset` bytes into a larger buffer, as a video sliced out of a decoder's buffer may."""
    host = np.random.default_rng(seed).integers(0, 256, (F, H, W, 3), dtype=np.uint8)
    dev = torch.from_numpy(host).cuda()
    if offset:
        buf = torch.zeros(host.size + offset + 16, dtype=torch.uint8, device="cuda")
        view = buf[offset:offset + host.size].view(F, H, W, 3)
        view.copy_(dev)
        assert view.is_contiguous() and view.data_ptr() % 16 == offset % 16
        dev = view
    return host, dev


def _face(rng, H, W, lo=150, hi=900):
    """(h, w) of a face box: lo .. hi px a side, at most the frame"""
    return int(rng.integers(lo, min(hi, H) + 1)), int(rng.integers(lo, min(hi, W) + 1))


def _video_boxes(rng, F, H, W):
    """(frame, y1, y2, x1, x2) rows: face-sized boxes anywhere, on each edge and in each corner; the whole frame; 1 px
    wide and 1 px tall boxes (one on the right edge, one on the bottom edge); 8 x 900 and 900 x 8 slivers; and boxes
    below 96 px, which the crop upscales."""
    boxes = []

    def add(y1, h, x1, w):
        boxes.append((int(rng.integers(0, F)), y1, y1 + h, x1, x1 + w))

    def anywhere(h, w):
        add(int(rng.integers(0, H - h + 1)), h, int(rng.integers(0, W - w + 1)), w)

    for _ in range(3):
        anywhere(*_face(rng, H, W))
    h, w = _face(rng, H, W)
    add(0, h, int(rng.integers(0, W - w + 1)), w)              # top edge
    h, w = _face(rng, H, W)
    add(H - h, h, int(rng.integers(0, W - w + 1)), w)          # bottom edge
    h, w = _face(rng, H, W)
    add(int(rng.integers(0, H - h + 1)), h, 0, w)              # left edge
    h, w = _face(rng, H, W)
    add(int(rng.integers(0, H - h + 1)), h, W - w, w)          # right edge
    for top in (True, False):                                  # the corners
        for left in (True, False):
            h, w = _face(rng, H, W)
            add(0 if top else H - h, h, 0 if left else W - w, w)
    add(0, H, 0, W)                                            # the whole frame
    anywhere(300, 1)
    add(int(rng.integers(0, H - 300)), 300, W - 1, 1)          # 1 px wide on the right edge
    anywhere(1, 300)
    add(H - 1, 1, int(rng.integers(0, W - 300)), 300)          # 1 px tall on the bottom edge
    anywhere(8, 900)
    anywhere(min(900, H), 8)
    anywhere(60, 80)
    add(H - 95, 95, W - 97, 97)                                # 95 x 97 in the bottom-right corner
    add(0, 97, W - 95, 95)                                     # 97 x 95 in the top-right corner
    return np.asarray(boxes, dtype=np.int32)


def test_kernels_hash_to_opencv_digests_at_video_sizes(gen, golden_dir):
    """crop_resize (the box cropped out of its whole frame) and paste (into a canvas of the box's size) on the
    resize_video.json cases hash to cv2.resize's own output, with no cv2 on the machine."""
    for case in _video_gold(golden_dir):
        if case["kind"] == "crop":
            (H, W), (y1, y2, x1, x2) = case["frame"], case["box"]
            frame = torch.from_numpy(_gold_image(H, W, case["seed"])[None]).cuda()
            got = gen.crop_resize(frame, [[0, y1, y2, x1, x2]])[0]
        else:
            h, w = case["size"]
            canvas = torch.zeros((1, h, w, 3), dtype=torch.uint8, device="cuda")
            got = gen.paste(torch.from_numpy(_gold_image(96, 96, case["seed"])[None]).cuda(), canvas, [[0, 0, h, 0, w]])[0]
        assert _sha256(got.cpu().numpy()) == case["sha256"], case


@pytest.mark.parametrize("offset", [0, 7])
@pytest.mark.parametrize("H,W", SIZES)
def test_offline_kernels_bit_exact_at_video_sizes(gen, H, W, offset):
    """crop_resize == P.crop_resize_batch, paste == P.paste_batch, and infer_frames == P.paste_batch of infer_u8 of
    crop_resize, bit for bit: the two calls run the generator at the same N, so w2l_lipsync_frames_u8 is pinned end to
    end without a float tolerance."""
    F = 2
    rng = np.random.default_rng(H * 7 + W + offset)
    host, fr = _frames(F, H, W, seed=H + W + offset, offset=offset)
    boxes = _video_boxes(rng, F, H, W)
    N = boxes.shape[0]
    crops = gen.crop_resize(fr, boxes)
    assert np.array_equal(crops.cpu().numpy(), P.crop_resize_batch(host, boxes))
    pred = torch.from_numpy(rng.integers(0, 256, (N, 96, 96, 3), dtype=np.uint8)).cuda()
    got = gen.paste(pred, fr, boxes)
    pred_h = pred.cpu().numpy()
    for i in range(N):
        assert np.array_equal(got[i].cpu().numpy(), P.paste_batch(pred_h[i:i + 1], host, boxes[i:i + 1])[0]), boxes[i]
    mel = torch.rand((N, 1, 80, 16), generator=torch.Generator().manual_seed(H + offset)) * 8 - 4
    with torch.no_grad():
        got = gen.infer_frames(mel.cuda(), fr, boxes)
        pred_h = gen.infer_u8(mel.cuda(), crops).cpu().numpy()
    for i in range(N):
        assert np.array_equal(got[i].cpu().numpy(), P.paste_batch(pred_h[i:i + 1], host, boxes[i:i + 1])[0]), boxes[i]


def _face_rects(rng, F, H, W, lo=150, hi=900, corners=None):
    """F detector rects (x1, y1, x2, y2) of faces lo .. hi px wide, centred anywhere in the frame: those near an edge
    stick out of it and are clipped when the boxes are padded (face_boxes).  corners: {frame: (right, bottom)}, frames
    whose face sticks out past that corner of the frame (0: left / top, 1: right / bottom), so that their box reaches
    both edges."""
    out = []
    for j in range(F):
        w = int(rng.integers(lo, hi + 1))
        h = int(w * rng.uniform(1.0, 1.3))
        if corners and j in corners:
            right, bottom = corners[j]
            cx, cy = (W - w // 4 if right else w // 4), (H - h // 4 if bottom else h // 4)
        else:
            cx, cy = int(rng.integers(0, W)), int(rng.integers(0, H))
        out.append((cx - w // 2, cy - h // 2, cx - w // 2 + w, cy - h // 2 + h))
    return np.asarray(out, dtype=np.int64)


def _bottom_right(H, W, h, w):
    return (H - h, H, W - w, W)


# name: (F, H, W, byte offset of the video, seconds of audio, fps, session keywords besides frames and fps)
STREAMS = {
    "1080p box in the corner": (6, 1080, 1920, 0, 0.80, 25.0, lambda rng, F, H, W: dict(box=_bottom_right(H, W, 430, 390))),
    # smoothed over 5 frames: the first rows' boxes stay in the top-left corner
    "720p faces": (8, 720, 1280, 0, 0.90, 29.97002997,
                   lambda rng, F, H, W: dict(rects=_face_rects(rng, F, H, W, hi=700, corners={j: (0, 0) for j in range(5)}))),
    "4K faces": (4, 2160, 3840, 0, 0.36, 25.0,
                 lambda rng, F, H, W: dict(rects=_face_rects(rng, F, H, W, lo=300, corners={1: (1, 0)}), nosmooth=True)),
    # the odd sizes: their last 16-byte piece starts 2, 1 and 0 bytes into a pixel (piece index % 3) and holds 1, 11
    # and 3 bytes; every box or every other box ends at the frame's last pixel
    "1079x1917 unaligned": (6, 1079, 1917, 5, 0.70, 30.0,
                            lambda rng, F, H, W: dict(rects=_face_rects(rng, F, H, W, corners=dict.fromkeys((0, 2, 4), (1, 1))),
                                                      nosmooth=True)),
    "1079x1919": (2, 1079, 1919, 0, 0.50, 25.0, lambda rng, F, H, W: dict(box=_bottom_right(H, W, 200, 180))),
    "719x1279 unaligned": (2, 719, 1279, 3, 0.50, 25.0, lambda rng, F, H, W: dict(box=_bottom_right(H, W, 151, 149))),
}


def _stream_case(name, seed):
    F, H, W, offset, sec, fps, kw = STREAMS[name]
    rng = np.random.default_rng(seed)
    _, frames = _frames(F, H, W, seed=seed, offset=offset)
    wav = M.make_wav(int(sec * 16000) + 37 * seed, seed=seed, kind="mix")
    return frames, wav, fps, kw(rng, F, H, W)


def _check_stream_output(gen, got, frames, wav, fps, kw):
    """got == the offline composition bit for bit, and every output frame equals its source frame outside its box"""
    ref = _offline(gen, frames, wav, fps, **kw)
    assert got.shape == ref.shape
    assert torch.equal(got, ref)
    F, H, W = frames.shape[:3]
    rows = offline_rows(wav.shape[0], fps, F, H, W, rects=kw.get("rects"), nosmooth=kw.get("nosmooth", False),
                        box=kw.get("box"))
    assert rows.shape[0] == got.shape[0]
    for i, _, j, y1, y2, x1, x2 in rows:
        g = got[i].clone()
        g[y1:y2, x1:x2] = frames[j][y1:y2, x1:x2]
        assert torch.equal(g, frames[j]), (i, j, y1, y2, x1, x2)


@pytest.mark.parametrize("max_batch", [1, 4, 16])
def test_stream_group_at_video_sizes(gen, max_batch):
    """One server over sessions of six frame sizes.  At max_batch 1 each paste launch covers its one frame with 8 blocks
    per SM of 256 threads x 16 bytes (4.3 MB a pass on 132 SMs), so 1080p and 4K frames take several passes of the
    grid-stride loop; at 16 one launch mixes frame sizes, boxes, alignments and padding rows."""
    from wav2lip_b200.stream import LipSyncServer
    rng = np.random.default_rng(max_batch)
    srv = LipSyncServer(gen, max_batch=max_batch)
    run, cases = _Run(srv, rng), {}
    for k, name in enumerate(STREAMS):
        frames, wav, fps, kw = _stream_case(name, seed=k)
        sid = srv.open(frames, fps, **kw)
        cases[sid] = (name, frames, wav, fps, kw)
        run.add(sid, _pieces(rng, wav, "random"))
    while run.tick():
        pass
    for sid, (name, frames, wav, fps, kw) in cases.items():
        try:
            _check_stream_output(gen, run.result(sid), frames, wav, fps, kw)
        except AssertionError as e:
            raise AssertionError(f"{name}: {e}") from e
    srv.close()


@pytest.mark.parametrize("name", ["1080p box in the corner", "1079x1917 unaligned"])
def test_lone_session_at_video_sizes(gen, name):
    from wav2lip_b200.stream import LipSyncSession
    k = list(STREAMS).index(name)
    frames, wav, fps, kw = _stream_case(name, seed=k)
    s = LipSyncSession(gen, frames, fps, batch=3, **kw)
    outs = [s.push(p)[1] for p in _pieces(np.random.default_rng(k), wav, "640")] + [s.finish()[1]]
    s.close()
    _check_stream_output(gen, torch.cat(outs), frames, wav, fps, kw)
