"""Scope rows (f): the mel chunker (inference.py:231-240) and the fused uint8 batch assembly around the
generator call (inference.py:134-140, 259-265, 269).  CPU part: chunk counting (host logic in libw2l) against
the verbatim NumPy restatement.  GPU part: kernels against the oracle."""
import numpy as np
import pytest
import torch

from oracle import mel_oracle as M
from oracle import pipeline_oracle as P
from oracle import w2l_oracle as O


def test_mel_num_chunks_host_logic():
    from wav2lip_b200 import _lib
    L = _lib.get_lib()
    for fps in (25.0, 24.0, 30.0, 23.976, 29.97, 50.0, 12.5, 60.0):
        for F in (16, 17, 31, 32, 80, 81, 241, 1000, 10000, 12345):
            mel = np.zeros((80, F), dtype=np.float32)
            assert L.w2l_mel_num_chunks(F, fps) == len(P.mel_chunks(mel, fps)), (F, fps)
    assert L.w2l_mel_num_chunks(15, 25.0) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("fps", [25.0, 29.97, 24.0])
def test_mel_chunks_bit_exact(fps):
    from wav2lip_b200 import audio
    wav = M.make_wav(16000 * 3 + 77, seed=4, kind="mix")
    mel = M.melspectrogram(wav)
    ref = np.stack(P.mel_chunks(mel, fps))[:, None]            # (n,1,80,16)
    got = audio.mel_chunks(mel, fps)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref)                             # pure gather: bit-exact
    # device path: mel computed and chunked on the GPU without touching the host
    mel_dev = audio.melspectrogram(torch.from_numpy(wav).cuda())
    chunks_dev = audio.mel_chunks(mel_dev, fps)
    assert chunks_dev.is_cuda and tuple(chunks_dev.shape) == ref.shape
    assert np.abs(chunks_dev.cpu().numpy() - ref).max() <= 1e-4
    with pytest.raises(ValueError):
        audio.mel_chunks(np.zeros((80, 10), dtype=np.float32), fps)


@pytest.mark.gpu
def test_fused_u8_assembly_matches_reference_pipeline():
    """faces uint8 -> [mask | full]/255 -> generator -> *255 -> uint8, against the oracle running the reference's
    own NumPy lines + the fp32 CPU generator.  Integer output through a float pipeline: |diff| <= 1 LSB, and
    the large majority of bytes identical."""
    import ctypes as C
    from wav2lip_b200 import _lib
    from wav2lip_b200.models import Wav2Lip
    rng = np.random.RandomState(3)
    N = 5
    faces = rng.randint(0, 256, size=(N, 96, 96, 3), dtype=np.uint8)
    wav = M.make_wav(16000, seed=9, kind="noise")
    mels = P.mel_chunks(M.melspectrogram(wav), 25.0)[:N]
    mel_b, img_b = P.assemble_batch(faces, mels)
    sd = O.make_state_dict("generator", 0, init="default")
    with torch.no_grad():
        pred = O.generator_forward(sd, torch.from_numpy(mel_b), torch.from_numpy(img_b)).numpy()
    ref = P.postprocess(pred)
    g = Wav2Lip()
    g.load_state_dict(sd, strict=True)
    g = g.cuda().eval()
    with torch.no_grad():
        out = g.infer_u8(torch.from_numpy(mel_b).cuda(), torch.from_numpy(faces).cuda())
        # the fp32 call on the oracle-assembled batch must agree with the fused path as well
        y32 = g(torch.from_numpy(mel_b).cuda(), torch.from_numpy(img_b).cuda()).cpu().numpy()
    out = out.cpu().numpy()
    assert out.shape == ref.shape and out.dtype == np.uint8
    d = np.abs(out.astype(np.int16) - ref.astype(np.int16))
    assert d.max() <= 1
    assert (d == 0).mean() >= 0.98
    assert np.array_equal(out, P.postprocess(y32))              # fused assembly == explicit assembly, bit for bit
    # host-buffer variant (pipelined) gives the same bytes
    ctx = g._w2l_ctx
    out_h = np.empty_like(out)
    mel_h = np.ascontiguousarray(mel_b)
    _lib.check(ctx.lib.w2l_generator_forward_u8_host(ctx.h, mel_h.ctypes.data_as(C.c_void_p), faces.ctypes.data_as(C.c_void_p),
                                                     out_h.ctypes.data_as(C.c_void_p), N))
    assert np.array_equal(out_h, out)
    with pytest.raises(ValueError):
        g.infer_u8(torch.from_numpy(mel_b).cuda(), torch.zeros((N, 96, 96, 3), device="cuda"))


@pytest.mark.gpu
def test_inference_loop_end_to_end_matches_composed_oracle():
    """examples/lipsync_loop.py (melspectrogram -> mel_chunks -> infer_stream over uint8 crops) against the oracle
    composed the way inference.py:224-271 composes it: mel_oracle -> pipeline_oracle.mel_chunks -> assemble_batch ->
    generator -> postprocess.  uint8 output through a float pipeline: <= 1 LSB."""
    import importlib.util
    import os
    from wav2lip_b200.models import Wav2Lip
    spec = importlib.util.spec_from_file_location(
        "lipsync_loop", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "lipsync_loop.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    fps, batch = 25.0, 7                                   # 1.3 s of audio -> 33 frames -> batches 7,7,7,7,5
    wav = M.make_wav(int(16000 * 1.3), seed=21, kind="mix")
    rng = np.random.RandomState(5)
    crops = rng.randint(0, 256, size=(10, 96, 96, 3), dtype=np.uint8)    # fewer crops than frames: looped
    sd = O.make_state_dict("generator", 0, init="default")
    g = Wav2Lip()
    g.load_state_dict(sd, strict=True)
    g = g.cuda().eval()
    got = ex.lipsync(g, wav, crops, fps, batch)
    mels = P.mel_chunks(M.melspectrogram(wav), fps)
    assert got.shape == (len(mels), 96, 96, 3) and got.dtype == np.uint8
    idx = np.arange(len(mels)) % len(crops)
    mel_b, img_b = P.assemble_batch(crops[idx], mels)
    with torch.no_grad():
        pred = O.generator_forward(sd, torch.from_numpy(mel_b), torch.from_numpy(img_b)).numpy()
    ref = P.postprocess(pred)
    d = np.abs(got.astype(np.int16) - ref.astype(np.int16))
    assert d.max() <= 1 and (d == 0).mean() >= 0.98


# ---- scope row f2, the two cv2.resize calls and the paste (inference.py:126, :269-271) ----------------------------------------
def _resize_gold(golden_dir):
    import os
    return np.load(os.path.join(golden_dir, "resize.npz"))


def _gold_image(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def test_resize_oracle_is_pinned_to_opencv_goldens(golden_dir):
    """oracle/pipeline_oracle.resize_linear_u8 == cv2.resize (vectors made by cv2 itself, tests/golden/make_golden_resize.py)."""
    g = _resize_gold(golden_dir)
    for i, (sh, sw, dh, dw) in enumerate(g["cases"]):
        got = P.resize_linear_u8(_gold_image(sh, sw, 1000 + i), (dw, dh))
        assert np.array_equal(got, g[f"out{i}"]), (i, sh, sw, dh, dw)
    frames = np.random.default_rng(7).integers(0, 256, (2, 120, 160, 3), dtype=np.uint8)
    pred = np.random.default_rng(8).integers(0, 256, (3, 96, 96, 3), dtype=np.uint8)
    assert np.array_equal(P.crop_resize_batch(frames, g["boxes"]), g["crops"])
    assert np.array_equal(P.paste_batch(pred, frames, g["boxes"]), g["pasted"])


def test_resize_oracle_against_live_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for it in range(120):
        H, W, dh, dw = (int(v) for v in rng.integers(1, 260, 4))
        if it % 3 == 0:
            dh = dw = 96
        if it % 4 == 0:
            H = W = 96
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(P.resize_linear_u8(img, (dw, dh)), cv2.resize(img, (dw, dh))), (H, W, dh, dw)
    # video frames: crops of face-sized and edge boxes down to 96 x 96 (2 to 40x), and 96 x 96 pastes up to the box
    pred = rng.integers(0, 256, (96, 96, 3), dtype=np.uint8)
    for H, W in ((720, 1280), (1080, 1920), (2160, 3840), (1079, 1917)):
        frame = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        boxes = [(0, H, 0, W), (H - 1, H, 0, W), (0, H, W - 1, W)]
        for k in range(12):
            h, w = (int(v) for v in rng.integers(60, min(H, 900) + 1, 2))
            y1, x1 = (0, 0) if k % 4 == 0 else (H - h, W - w) if k % 4 == 1 else (int(rng.integers(0, H - h + 1)),
                                                                                  int(rng.integers(0, W - w + 1)))
            boxes.append((y1, y1 + h, x1, x1 + w))
        for y1, y2, x1, x2 in boxes:
            crop = frame[y1:y2, x1:x2]
            assert np.array_equal(P.resize_linear_u8(crop, (96, 96)), cv2.resize(crop, (96, 96))), (H, W, y1, y2, x1, x2)
            if (y2 - y1) * (x2 - x1) <= 1200 * 1200:       # the whole-frame pastes are in resize_video.json
                assert np.array_equal(P.resize_linear_u8(pred, (x2 - x1, y2 - y1)), cv2.resize(pred, (x2 - x1, y2 - y1))), \
                    (H, W, y1, y2, x1, x2)


def _video_gold(golden_dir):
    import json
    import os
    with open(os.path.join(golden_dir, "resize_video.json")) as f:
        return json.load(f)["cases"]


def _video_gold_output(case, resize):
    """resize(src, dsize) on the seeded source of one resize_video.json case (tests/golden/make_golden_resize.py)"""
    if case["kind"] == "crop":
        (H, W), (y1, y2, x1, x2) = case["frame"], case["box"]
        return resize(_gold_image(H, W, case["seed"])[y1:y2, x1:x2], (96, 96))
    h, w = case["size"]
    return resize(_gold_image(96, 96, case["seed"]), (w, h))


def _sha256(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


def test_resize_oracle_is_pinned_to_opencv_digests_at_video_sizes(golden_dir):
    """The oracle's crops and pastes at 720p, 1080p, 4K and 1079 x 1917 hash to the SHA-256 of cv2.resize's output
    (tests/golden/resize_video.json, made by cv2 itself)."""
    cases = _video_gold(golden_dir)
    assert len(cases) >= 20
    for case in cases:
        assert _sha256(_video_gold_output(case, P.resize_linear_u8)) == case["sha256"], case


@pytest.mark.gpu
def test_crop_resize_and_paste_bit_exact_with_opencv(golden_dir):
    from wav2lip_b200 import _lib
    from wav2lip_b200.models import Wav2Lip
    g = _resize_gold(golden_dir)
    frames = np.random.default_rng(7).integers(0, 256, (2, 120, 160, 3), dtype=np.uint8)
    pred = np.random.default_rng(8).integers(0, 256, (3, 96, 96, 3), dtype=np.uint8)
    m = Wav2Lip().cuda().eval()
    fr = torch.from_numpy(frames).cuda()
    crops = m.crop_resize(fr, g["boxes"]).cpu().numpy()
    assert np.array_equal(crops, g["crops"])                       # == cv2.resize, bit for bit
    pasted = m.paste(torch.from_numpy(pred).cuda(), fr, g["boxes"]).cpu().numpy()
    assert np.array_equal(pasted, g["pasted"])
    # every golden case as a crop (sources up to 300 px) and as a paste target
    for i, (sh, sw, dh, dw) in enumerate(g["cases"]):
        img = _gold_image(sh, sw, 1000 + i)
        if (dh, dw) == (96, 96):
            got = m.crop_resize(torch.from_numpy(img[None]).cuda(), [[0, 0, sh, 0, sw]]).cpu().numpy()[0]
            assert np.array_equal(got, g[f"out{i}"]), i
        if (sh, sw) == (96, 96):
            canvas = np.zeros((1, dh + 3, dw + 2, 3), dtype=np.uint8)
            got = m.paste(torch.from_numpy(img[None]).cuda(), torch.from_numpy(canvas).cuda(), [[0, 3, dh + 3, 1, dw + 1]]).cpu().numpy()[0]
            assert np.array_equal(got[3:, 1:dw + 1], g[f"out{i}"]), i
            assert got[:3].max() == 0 and got[:, 0].max() == 0 and got[:, dw + 1:].max() == 0
    # random boxes against the oracle at a video-like frame size
    rng = np.random.default_rng(5)
    frames = rng.integers(0, 256, (3, 270, 480, 3), dtype=np.uint8)
    boxes = []
    for _ in range(9):
        y1, x1 = int(rng.integers(0, 150)), int(rng.integers(0, 300))
        boxes.append([int(rng.integers(0, 3)), y1, y1 + int(rng.integers(20, 120)), x1, x1 + int(rng.integers(20, 180))])
    fr = torch.from_numpy(frames).cuda()
    assert np.array_equal(m.crop_resize(fr, boxes).cpu().numpy(), P.crop_resize_batch(frames, boxes))
    with pytest.raises(_lib.W2LError):
        m.crop_resize(fr, [[0, 10, 10, 0, 5]])                     # empty box
    with pytest.raises(_lib.W2LError):
        m.crop_resize(fr, [[3, 0, 10, 0, 5]])                      # frame index out of range


@pytest.mark.gpu
def test_infer_frames_equals_the_composed_inner_loop():
    """inference.py:120-140 + :259-271 in one call == crop/resize -> assemble -> generator -> x255 -> uint8 -> resize -> paste
    composed from the oracle pieces; the generator runs in fp16 on the GPU, so predictions may differ by one grey level
    before the final resize: pasted pixels within 1 LSB, everything outside the boxes bit-identical."""
    from wav2lip_b200.models import Wav2Lip
    sd = O.make_state_dict("generator", 0)
    m = Wav2Lip()
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    rng = np.random.default_rng(11)
    frames = rng.integers(0, 256, (2, 144, 176, 3), dtype=np.uint8)
    boxes = np.array([[0, 20, 130, 30, 150], [1, 0, 96, 40, 136], [0, 44, 100, 10, 90]], dtype=np.int32)
    mel = (torch.rand((3, 1, 80, 16), generator=torch.Generator().manual_seed(2)) * 8 - 4)
    with torch.no_grad():
        got = m.infer_frames(mel.cuda(), torch.from_numpy(frames).cuda(), boxes).cpu().numpy()
        crops = P.crop_resize_batch(frames, boxes)
        mel_b, img_b = P.assemble_batch(crops, [x[0].numpy() for x in mel])
        pred = O.generator_forward(sd, torch.from_numpy(mel_b), torch.from_numpy(img_b)).numpy()
    ref = P.paste_batch(P.postprocess(pred), frames, boxes)
    assert got.shape == ref.shape == (3, 144, 176, 3)
    d = np.abs(got.astype(int) - ref.astype(int))
    assert d.max() <= 2, d.max()          # stress weights: a borderline prediction may round to the neighbouring grey level twice
    assert (d > 0).mean() <= 0.05
    for i, (f, y1, y2, x1, x2) in enumerate(boxes):
        mask = np.ones((144, 176), dtype=bool)
        mask[y1:y2, x1:x2] = False
        assert np.array_equal(got[i][mask], frames[f][mask])
