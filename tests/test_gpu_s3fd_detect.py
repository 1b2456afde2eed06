"""The S3FD detector on the device (`w2l_s3fd_detect_u8`, `SFDDetector.detect_from_batch_u8`,
`FaceAlignment.get_detections_for_batch_u8`): uint8 frames in, boxes out.

What is checked, and against what:
- Ingest: the 12 maps of a detection call are bit-identical to `w2l_s3fd_forward` on `preprocess(frames)` (the mean-
  subtracted values are integers, exact in fp16 / bf16), with and without the channel reversal, at 96x128, 150x210 and
  16 x 720x1280.
- Select / decode, against float64 on the GPU's own maps.  Score bar: the softmax is e1 / (e0 + e1) with e_k =
  expf(x_k - max); expf is within 2 ulp, the subtraction, the add and the division round once each, and the rounding of
  d = x1 - x0 moves p by p(1-p)|d| 2^-24: bar_p = 2^-24 (12 p + 2 p (1-p) |d|).  Box bar: A = 4 * stride is a power of
  two (exact products), loc * 0.1f and loc * 0.2f round once, expf within 2 ulp, the adds round once:
  e(cx) = 2^-24 (A |t0| + |cx|), e(w) = 2^-24 |w| (|t2| + 5), e(x1) = e(cx) + e(w)/2 + 2^-24 |x1|,
  e(x2) = e(w) + e(x1) + 2^-24 |x2| (t0 = loc0 * 0.1f, t2 = loc2 * 0.2f; the same for y).  The candidate set is
  {p64 > 0.5} except locations within bar_p of 0.5.
- Sort and NMS, bit for bit: a NumPy restatement of bbox.py:44-64 in float32 (NumPy rounds every op and never contracts)
  with the tie rule np.argsort(s, kind="stable")[::-1], on the device's own candidates, at max_det = all, 1 and 3.
- Constructed ties (zero head weights; the conf biases pass one or two scales with one identical score; loc biases zero,
  a uniform centre shift, or w/h channels whose expf overflows to NaN boxes): the whole output equals the closed-form NMS of
  the anchor grid bit for bit, on both NMS paths (shared memory, and global memory above kNmsSmemCap = 4096 candidates).
- Against the reference: the oracle's `detect_from_batch` at the tolerance of test_detector_end_to_end_vs_oracle; and
  `get_detections_for_batch_u8` against `get_detections_for_batch` on the same frames, which differ only through host vs
  device exp and the host path's float64 centre: a different first box is allowed only where the top score is within
  the score bar of the runner-up or of 0.5, a coordinate only by 1 where its float value is within the box bar of an
  integer.
- Batch independence, determinism, empty images and argument checks.

Measured on one H100 80GB HBM3 (700 W), make_state_dict(0), max err / bar over all candidates:
  2 x 96x128 (246 / 248 candidates, shared-memory NMS)     scores 0.163, boxes 0.570
  1 x 150x210 (583 candidates, shared-memory NMS)          scores 0.155, boxes 0.654
  16 x 720x1280 (~18.3 k candidates each, global NMS)      scores 0.183, boxes 0.938
- An FMA-contracted overlap denominator moves an overlap by one ulp, which changes a decision only within an ulp of 0.3:
  test_nms_rounds_the_overlap_denominator uses uniform non-integer anchor widths chosen so that it does.
Deliberate defects caught by this file: an FMA-contracted IoU denominator, fma(-w, h, area_i + area_j) (the FMA-sensitive
grids: 144 boxes kept instead of 146), suppression written as ovr > 0.3 (the NaN-box case), ties ordered by ascending
location, the scale-0 max-out dropped (720p candidate set; the constructed cases put the max in channel 2), and a
compaction that orders the warps of a chunk backwards.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import s3fd_oracle as S

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TAPS = ["conv3_3_norm", "conv4_3_norm", "conv5_3_norm", "fc7", "conv6_2", "conv7_2"]


def _net(sd):
    from wav2lip_b200.face_detection.detection.sfd.net_s3fd import s3fd
    m = s3fd()
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def net():
    return _net(S.make_state_dict(0))


def _detect(net, frames, max_det, reverse=False, maps=False):
    with torch.no_grad():
        d, c, o = net.detect_u8(torch.from_numpy(frames).cuda(), max_det, reverse_channels=reverse, return_maps=maps)
    torch.cuda.synchronize()
    return d.cpu().numpy(), c.cpu().numpy(), (None if o is None else [t.cpu().numpy() for t in o])


def _forward_maps(net, bgr):
    with torch.no_grad():
        return [t.cpu().numpy() for t in net(S.preprocess(bgr).cuda())]


def _decode64(maps):
    """Per location (scale-major, row, column): p64, bar_p, box64 (4), box bar (4) in float64 from the float32 maps."""
    P, BP, BX, BB = [], [], [], []
    f = np.float64
    for i in range(6):
        cls, reg = maps[2 * i].astype(f), maps[2 * i + 1]
        B, _, h, w = cls.shape
        d = cls[:, 1] - cls[:, 0]
        p = 1.0 / (1.0 + np.exp(-d))
        stride = 4 << i
        A = f(4 * stride)
        yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        axc, ayc = stride / 2 + xx * stride, stride / 2 + yy * stride
        t0 = (reg[:, 0] * np.float32(0.1)).astype(f)     # the float32 products the device rounds, exactly
        t1 = (reg[:, 1] * np.float32(0.1)).astype(f)
        t2 = reg[:, 2].astype(f) * f(np.float32(0.2))
        t3 = reg[:, 3].astype(f) * f(np.float32(0.2))
        with np.errstate(over="ignore", invalid="ignore"):
            cx, cy = axc + t0 * A, ayc + t1 * A
            ww, hh = A * np.exp(t2), A * np.exp(t3)
            x1, y1 = cx - ww / 2, cy - hh / 2
            x2, y2 = x1 + ww, y1 + hh
            ecx, ecy = U * (A * np.abs(t0) + np.abs(cx)), U * (A * np.abs(t1) + np.abs(cy))
            ew, eh = U * ww * (np.abs(t2) + 5), U * hh * (np.abs(t3) + 5)
            ex1, ey1 = ecx + ew / 2 + U * np.abs(x1), ecy + eh / 2 + U * np.abs(y1)
            ex2, ey2 = ew + ex1 + U * np.abs(x2), eh + ey1 + U * np.abs(y2)
        P.append(p.reshape(B, -1))
        BP.append((U * (12 * p + 2 * p * (1 - p) * np.abs(d))).reshape(B, -1))
        BX.append(np.stack([x1, y1, x2, y2], -1).reshape(B, -1, 4))
        BB.append(np.stack([ex1, ey1, ex2, ey2], -1).reshape(B, -1, 4))
    return (np.concatenate(P, 1), np.concatenate(BP, 1), np.concatenate(BX, 1), np.concatenate(BB, 1))


def _nms32(c, max_det, fma=False):
    """bbox.py:44-64 in float32 on candidates already in the tie-rule order; returns the kept row indices.  fma: the
    denominator contracted as fma(-w, h, area_i + area_j) (float64 holds w*h exactly), the arithmetic the device must
    NOT use."""
    x1, y1, x2, y2 = (c[:, k].astype(np.float32) for k in range(4))
    one, zero, thr = np.float32(1), np.float32(0), np.float32(0.3)
    with np.errstate(invalid="ignore", over="ignore"):
        areas = (x2 - x1 + one) * (y2 - y1 + one)
        order = np.arange(len(c))
        keep = []
        while order.size > 0 and len(keep) < max_det:
            i = order[0]
            keep.append(i)
            r = order[1:]
            xx1, yy1 = np.maximum(x1[i], x1[r]), np.maximum(y1[i], y1[r])
            xx2, yy2 = np.minimum(x2[i], x2[r]), np.minimum(y2[i], y2[r])
            w, h = np.maximum(zero, xx2 - xx1 + one), np.maximum(zero, yy2 - yy1 + one)
            if fma:
                den = ((areas[i] + areas[r]).astype(np.float64) - w.astype(np.float64) * h.astype(np.float64)).astype(np.float32)
                ovr = w * h / den
            else:
                ovr = w * h / (areas[i] + areas[r] - w * h)
            order = r[ovr <= thr]
    return keep


def _tie_order(scores):
    return np.argsort(scores, kind="stable")[::-1]


def _same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(
        np.where(np.isnan(a), 0, a).view(np.uint32), np.where(np.isnan(b), 0, b).view(np.uint32))


# ---- 1. ingest -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,reverse", [(2, 96, 128, False), (2, 96, 128, True), (1, 150, 210, False),
                                           (1, 150, 210, True), (16, 720, 1280, True)])
def test_maps_bit_identical_to_float_path(net, B, H, W, reverse):
    frames = S.make_images(B, H, W, seed=3)
    _, _, maps = _detect(net, frames, 1, reverse=reverse, maps=True)
    ref = _forward_maps(net, np.ascontiguousarray(frames[..., ::-1]) if reverse else frames)
    for i, (a, b) in enumerate(zip(maps, ref)):
        assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), i


# ---- 2./3. select, decode, sort, NMS on the GPU's own maps ---------------------------------------------------------------
@pytest.mark.parametrize("B,H,W", [(2, 96, 128), (1, 150, 210), (16, 720, 1280)])
def test_candidates_vs_float64_and_nms_bit_exact(net, B, H, W):
    frames = S.make_images(B, H, W, seed=5)
    L = net.num_anchors(H, W)
    by_md = {md: _detect(net, frames, md)[:2] for md in (1, 3)}
    dets, counts, maps = _detect(net, frames, L, maps=True)
    by_md[L] = (dets, counts)
    p64, bp, bx, bb = _decode64(maps)
    ctx = net._w2l_ctx
    worst_s = worst_b = 0.0
    paths = set()
    for b in range(B):
        cand, path = ctx.s3fd_candidates(b)
        paths.add(path)
        loc = cand[:, 5].astype(np.int64)
        sure = np.abs(p64[b] - 0.5) > bp[b]
        want = set(np.nonzero(sure & (p64[b] > 0.5))[0])
        got = set(loc.tolist())
        assert want <= got and not (got - want) - set(np.nonzero(~sure)[0]), b
        es = np.abs(cand[:, 4].astype(np.float64) - p64[b, loc]) / bp[b, loc]
        eb = np.abs(cand[:, :4].astype(np.float64) - bx[b, loc]) / bb[b, loc]
        worst_s, worst_b = max(worst_s, es.max(initial=0)), max(worst_b, np.nanmax(eb, initial=0))
        assert np.all(es <= 1.0), (b, es.max())
        assert np.all(eb <= 1.0), (b, eb.max())
        # sorted by score, ties by descending location: exactly the stable argsort reversed of the location-ordered list
        by_loc = cand[np.argsort(loc)]
        assert np.array_equal(by_loc[_tie_order(by_loc[:, 4])], cand), b
        for md, (d, c) in by_md.items():
            keep = _nms32(cand, md)
            assert c[b] == len(keep), (b, md, c[b], len(keep))
            assert _same_bits(d[b, :c[b]], cand[keep, :5]), (b, md)
            assert not d[b, c[b]:].any()
    print(f"[{B}x{H}x{W}] candidates/image {[int(ctx.s3fd_candidates(b)[0].shape[0]) for b in range(B)]}, "
          f"nms paths {sorted(paths)}, score err/bar {worst_s:.3f}, box err/bar {worst_b:.3f}")


# ---- 4. constructed ties ---------------------------------------------------------------------------------------------------
def _tie_state(pass_scales, loc):
    sd = S.make_state_dict(0)
    for i, t in enumerate(TAPS):
        for kind in ("conf", "loc"):
            sd[f"{t}_mbox_{kind}.weight"].zero_()
        conf = sd[f"{t}_mbox_conf.bias"]
        if i == 0:   # the background logit is the max of channels 0-2 (net_s3fd.py:123-126): put it in channel 2
            conf[:] = torch.tensor([-1.0, -3.0, 0.0, 2.0] if i in pass_scales else [-5.0, 0.0, 5.0, 0.0])
        else:
            conf[:] = torch.tensor([0.0, 2.0] if i in pass_scales else [5.0, 0.0])
        sd[f"{t}_mbox_loc.bias"][:] = torch.tensor(loc)
    return sd


def _closed_form(H, W, pass_scales, loc, score):
    """The anchor grid's candidates in location order, decoded in float32 as the reference does."""
    dims = (C.c_int32 * 12)()
    from wav2lip_b200 import _lib
    _lib.check(_lib.get_lib().w2l_s3fd_out_dims(H, W, dims))
    f = np.float32
    rows = []
    with np.errstate(over="ignore", invalid="ignore"):
        for i in range(6):
            h, w = dims[2 * i], dims[2 * i + 1]
            if i not in pass_scales:
                continue
            s = 4 << i
            A = f(4 * s)
            yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
            axc, ayc = (s / 2 + xx * s).astype(f).ravel(), (s / 2 + yy * s).astype(f).ravel()
            cx, cy = axc + (f(loc[0]) * f(0.1)) * A, ayc + (f(loc[1]) * f(0.1)) * A
            bw, bh = A * np.exp(f(loc[2]) * f(0.2)), A * np.exp(f(loc[3]) * f(0.2))
            x1, y1 = cx - bw / f(2), cy - bh / f(2)
            rows.append(np.stack([x1, y1, bw + x1, bh + y1, np.full_like(x1, score)], 1))
    return np.concatenate(rows).astype(np.float32)


@pytest.mark.parametrize("H,W,pass_scales,loc,path", [
    (128, 128, (0,), (0.0, 0.0, 0.0, 0.0), 0),
    (128, 160, (1, 2), (0.37, -0.61, 0.0, 0.0), 0),
    (256, 256, (0, 1), (0.0, 0.0, 0.0, 0.0), 1),          # 4096 + 1024 candidates: above the shared-memory cap
    (256, 256, (0, 1), (0.37, -0.61, 0.0, 0.0), 1),
    (128, 128, (0, 2), (0.0, 0.0, 500.0, 500.0), 0),       # expf overflows: NaN boxes, the first one suppresses the rest
])
def test_constructed_ties_closed_form(H, W, pass_scales, loc, path):
    net = _net(_tie_state(pass_scales, loc))
    frames = S.make_images(2, H, W, seed=7)
    L = net.num_anchors(H, W)
    dets, counts, _ = _detect(net, frames, L)
    cand0, got_path = net._w2l_ctx.s3fd_candidates(0)
    assert got_path == path
    score = cand0[0, 4]   # one identical score everywhere (expf of the bias difference is the device's own)
    assert np.all(cand0[:, 4] == score) and abs(float(score) - 1 / (1 + np.exp(-2.0))) < 1e-6
    ref = _closed_form(H, W, pass_scales, loc, score)
    ref = ref[_tie_order(ref[:, 4])]
    assert _same_bits(cand0[:, :5], ref)
    keep = _nms32(ref, L)
    for b in range(2):
        assert counts[b] == len(keep), (b, counts[b], len(keep))
        assert _same_bits(dets[b, :counts[b]], ref[keep]), b
    if loc[2] > 100:
        assert counts[0] == 1 and np.isnan(dets[0, 0, 2])


# w/h loc biases (c2, c3) that put some anchor pair of the 16 x 16 stride-4 grid of a 64 x 64 image at an overlap whose
# rounded and FMA-contracted denominators fall on opposite sides of 0.3, so that the keep lists differ.  Found on the host
# by bisecting c2 to the adjacent-anchor crossing (w + 1 - 4) / (w + 1 + 4) = 0.3 and scanning c3 and the nearest float32
# values of c2 with the emulation in _nms32.  The widths are A * expf(0.2 c): not integers, so w * h rounds.
FMA_CASES = [(-4.559181213378906, -4.9604268074035645), (-4.559183120727539, -5.418053150177002),
             (-4.559181213378906, -5.466944694519043), (-4.559181213378906, -5.494523048400879),
             (-4.559181213378906, -5.432828903198242), (-4.559181213378906, -4.900576114654541)]


def test_nms_rounds_the_overlap_denominator():
    """The device NMS equals the rounded restatement on grids where an FMA-contracted denominator changes the result."""
    sensitive = 0
    for c2, c3 in FMA_CASES:
        net = _net(_tie_state((0,), (0.0, 0.0, c2, c3)))
        frames = S.make_images(1, 64, 64, seed=17)
        dets, counts, _ = _detect(net, frames, 1024)
        cand, path = net._w2l_ctx.s3fd_candidates(0)
        assert path == 0 and len(cand) == 256
        keep = _nms32(cand, 1024)
        assert counts[0] == len(keep) and _same_bits(dets[0, :counts[0]], cand[keep, :5]), (c2, c3)
        sensitive += _nms32(cand, 1024, fma=True) != keep
    # the cases only test something if the device's own boxes (its expf) reproduce the borderline pair
    assert sensitive >= 1, sensitive


def _raise_bg(sd, bg):
    for i, t in enumerate(TAPS):
        b = sd[f"{t}_mbox_conf.bias"]
        if i == 0:
            b[:3] += bg
        else:
            b[0] += bg
    return sd


# ---- 5. against the reference ----------------------------------------------------------------------------------------------
def test_detect_vs_oracle(net):
    sd = S.make_state_dict(0)
    imgs_bgr = S.make_images(2, 96, 128, seed=1)
    from wav2lip_b200.face_detection.detection.sfd.sfd_detector import SFDDetector
    det = SFDDetector.__new__(SFDDetector)
    det.device, det.verbose, det.face_detector = "cuda", False, net
    got = det.detect_from_batch_u8(imgs_bgr)
    ref = S.detect_from_batch(sd, imgs_bgr)
    for g, r in zip(got, ref):
        assert g.dtype == np.float32 and g.ndim == 2 and g.shape[1] == 5
        assert abs(len(g) - len(r)) <= max(3, 0.05 * len(r)), (len(g), len(r))
        if len(r):
            gb, rb = g[:, :4].astype(np.float64), np.array(r)[:, :4].astype(np.float64)
            d = (np.abs(gb[:, None, :] - rb[None, :, :]).max(axis=2) / (1.0 + np.abs(gb).max(axis=1))[:, None]).min(axis=1)
            assert np.mean(d <= 2e-2) >= 0.9, np.mean(d <= 2e-2)
    # device-resident frames give the same result as host frames
    got_dev = det.detect_from_batch_u8(torch.from_numpy(imgs_bgr).cuda())
    assert all(_same_bits(a, b) for a, b in zip(got, got_dev))


@pytest.mark.parametrize("B,H,W,bg", [(4, 240, 320, 0.0), (16, 720, 1280, 5.0)])
def test_get_detections_u8_matches_host_path(net, B, H, W, bg):
    """bg raises the conf heads' background bias: at 720p random weights pass ~18 k locations per image, which the host
    path's O(n^2) NMS takes minutes over."""
    from wav2lip_b200.face_detection import FaceAlignment, LandmarksType
    fa = FaceAlignment(LandmarksType._2D, flip_input=False, device="cuda")
    if bg:
        net = _net(_raise_bg(S.make_state_dict(0), bg))
    fa.face_detector.face_detector = net
    rgb = S.make_images(B, H, W, seed=11)
    host = fa.get_detections_for_batch(rgb)
    dev = fa.get_detections_for_batch_u8(rgb)
    assert len(host) == len(dev) == B
    _, _, maps = _detect(net, rgb, 1, reverse=True, maps=True)
    p64, bp, bx, bb = _decode64(maps)
    print(f"[{B}x{H}x{W}] images with a face: {sum(r is not None for r in host)} host, {sum(r is not None for r in dev)} device")
    for b in range(B):
        if host[b] == dev[b]:
            continue
        order = np.argsort(-p64[b], kind="stable")
        top, second = order[0], order[1]
        near = (abs(p64[b, top] - p64[b, second]) <= bp[b, top] + bp[b, second] or abs(p64[b, top] - 0.5) <= bp[b, top])
        if near:
            continue
        assert host[b] is not None and dev[b] is not None, b
        fl = np.maximum(bx[b, top], 0)
        for k in range(4):
            if host[b][k] != dev[b][k]:
                assert abs(host[b][k] - dev[b][k]) == 1, (b, host[b], dev[b])
                assert abs(fl[k] - np.round(fl[k])) <= bb[b, top, k] + U * abs(fl[k]), (b, k, fl[k])


# ---- 6. batch independence, determinism, empty images, argument checks ------------------------------------------------------
def test_batch_independence_and_determinism(net):
    frames = S.make_images(4, 150, 210, seed=13)
    L = net.num_anchors(150, 210)
    d4, c4, m4 = _detect(net, frames, L, maps=True)
    d4b, c4b, m4b = _detect(net, frames, L, maps=True)
    assert np.array_equal(c4, c4b) and _same_bits(d4, d4b)
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(m4, m4b))
    for b in range(4):
        d1, c1, m1 = _detect(net, frames[b:b + 1], L, maps=True)
        for a, m in zip(m1, m4):
            assert np.array_equal(a[0].view(np.uint32), m[b].view(np.uint32)), b
        assert c1[0] == c4[b] and _same_bits(d1[0], d4[b]), b


def test_no_candidate_gives_none_and_zero_count():
    net = _net(_tie_state((), (0.0, 0.0, 0.0, 0.0)))
    from wav2lip_b200.face_detection import FaceAlignment, LandmarksType
    fa = FaceAlignment(LandmarksType._2D, flip_input=False, device="cuda")
    fa.face_detector.face_detector = net
    rgb = S.make_images(3, 96, 128, seed=2)
    assert fa.get_detections_for_batch_u8(rgb) == [None, None, None]
    d, c, _ = _detect(net, rgb, 4)
    assert not c.any() and not d.any()


def test_invalid_arguments_raise_before_launch(net):
    from wav2lip_b200 import _lib
    frames = torch.from_numpy(S.make_images(1, 96, 128)).cuda()
    net.detect_u8(frames, 1)
    torch.cuda.synchronize()
    ctx = net._w2l_ctx
    n0 = ctx.launch_count()
    with pytest.raises(TypeError):
        net.detect_u8(frames.float(), 1)
    for bad in (frames[..., :2], frames[:, :31], frames[0]):
        with pytest.raises(ValueError):
            net.detect_u8(bad, 1)
    for md in (0, -1, 1.5, True):
        with pytest.raises(ValueError):
            net.detect_u8(frames, md)
    from wav2lip_b200.face_detection.detection.sfd.sfd_detector import SFDDetector
    det = SFDDetector.__new__(SFDDetector)
    det.device, det.verbose, det.face_detector = "cuda", False, net
    with pytest.raises(TypeError):
        det.detect_from_batch_u8(np.zeros((1, 96, 128, 3), np.float32))
    with pytest.raises(ValueError):
        det.detect_from_batch_u8(np.zeros((1, 96, 128, 4), np.uint8))
    out = torch.zeros((1, 1, 5), device="cuda")
    cnt = torch.zeros((1,), device="cuda", dtype=torch.int32)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    for args in ((1, 96, 128, 0, 0), (0, 96, 128, 0, 1), (1, 31, 128, 0, 1), (1, 96, 128, 2, 1)):
        B, H, W, rev, md = args
        assert ctx.lib.w2l_s3fd_detect_u8(ctx.h, p(frames), B, H, W, rev, md, p(out), p(cnt), None, None) == _lib.W2L_EINVAL
    assert ctx.launch_count() == n0
