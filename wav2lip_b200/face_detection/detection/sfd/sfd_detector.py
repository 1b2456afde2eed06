"""The detector around the network (face_detection/detection/sfd/sfd_detector.py:17-49, detect.py:58-94, bbox.py:44-64 of the
reference), host side: softmax of the class maps, the 0.05 candidate threshold, prior decoding with variances (0.1, 0.2),
greedy NMS at IoU 0.3 and the final 0.5 score cut — vectorised NumPy with the reference's semantics, including its batch
quirk: a location that passes the threshold in ANY image of the batch becomes a candidate in EVERY image (detect.py:77-88)."""
import os

import numpy as np
import torch

from .net_s3fd import s3fd

MEAN_BGR = np.array([104.0, 117.0, 123.0])


def decode_candidates(olist, thresh=0.05):
    """olist: the 12 maps as float32 numpy arrays.  Returns (n_candidates, B, 5) = x1, y1, x2, y2, score — the array
    batch_detect builds (detect.py:66-93)."""
    B = olist[0].shape[0]
    rows = []
    for i in range(6):
        cls, reg = olist[2 * i], olist[2 * i + 1]
        e = np.exp(cls - cls.max(axis=1, keepdims=True))
        prob = e[:, 1] / e.sum(axis=1)                                       # F.softmax(cls, dim=1)[:, 1]
        stride = 2 ** (i + 2)
        _, hh, ww = np.where(prob > thresh)                                  # one candidate per (image, y, x) hit, as the reference's zip
        if hh.size == 0:
            continue
        axc, ayc = stride / 2 + ww * stride, stride / 2 + hh * stride
        loc = reg[:, :, hh, ww]                                               # (B, 4, n)
        cx = axc[None] + loc[:, 0] * 0.1 * (stride * 4)
        cy = ayc[None] + loc[:, 1] * 0.1 * (stride * 4)
        w = stride * 4 * np.exp(loc[:, 2] * 0.2)
        h = stride * 4 * np.exp(loc[:, 3] * 0.2)
        x1, y1 = cx - w / 2, cy - h / 2
        box = np.stack([x1, y1, x1 + w, y1 + h, prob[:, hh, ww]], axis=2)    # (B, n, 5)
        rows.append(np.transpose(box, (1, 0, 2)))
    if not rows:
        return np.zeros((1, B, 5))
    return np.concatenate(rows, axis=0).astype(np.float32)


def nms(dets, thresh):
    """Greedy NMS of bbox.py:44-64 (boxes with +1 pixel extents, descending score, keep while overlap <= thresh)."""
    if len(dets) == 0:
        return []
    x1, y1, x2, y2, sc = dets[:, 0], dets[:, 1], dets[:, 2], dets[:, 3], dets[:, 4]
    area = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = sc.argsort()[::-1]
    keep = []
    while order.size > 0:
        i, rest = order[0], order[1:]
        keep.append(i)
        iw = np.maximum(0.0, np.minimum(x2[i], x2[rest]) - np.maximum(x1[i], x1[rest]) + 1)
        ih = np.maximum(0.0, np.minimum(y2[i], y2[rest]) - np.maximum(y1[i], y1[rest]) + 1)
        ovr = iw * ih / (area[i] + area[rest] - iw * ih)
        order = rest[ovr <= thresh]
    return keep


class SFDDetector:
    def __init__(self, device="cuda", path_to_detector=None, verbose=False):
        self.device, self.verbose = device, verbose
        self.face_detector = s3fd()
        path = path_to_detector or os.path.join(os.path.dirname(os.path.abspath(__file__)), "s3fd.pth")
        if os.path.isfile(path):
            self.face_detector.load_state_dict(torch.load(path, map_location="cpu"))
        elif path_to_detector is not None:
            raise FileNotFoundError(path_to_detector)
        # (no network access here: without s3fd.pth the detector keeps its random initialisation; the reference downloads it)
        self.face_detector.to(device)
        self.face_detector.eval()

    def detect_from_batch(self, images):
        """images (B,H,W,3) uint8 BGR -> per image a list of [x1, y1, x2, y2, score] rows (sfd_detector.py:40-46)."""
        imgs = np.asarray(images).astype(np.float32) - MEAN_BGR.astype(np.float32)
        x = torch.from_numpy(np.ascontiguousarray(imgs.transpose(0, 3, 1, 2))).to(self.device)
        with torch.no_grad():
            olist = [o.cpu().numpy() for o in self.face_detector(x)]
        cand = decode_candidates(olist)
        out = []
        for i in range(cand.shape[1]):
            d = cand[:, i, :]
            d = d[nms(d, 0.3), :]
            out.append([r for r in d if r[-1] > 0.5])
        return out

    def detect_from_batch_u8(self, images, max_det=None, reverse_channels=False):
        """`detect_from_batch` on the device: images (B,H,W,3) uint8 BGR, a CUDA tensor or host memory (copied to the
        device once, as uint8) -> per image a float32 (k, 5) array of x1, y1, x2, y2, score, best first, at most max_det
        rows (None: every box).  The content is `detect_from_batch`'s, up to the order of exactly tied scores (the larger
        location index first, DESIGN.md §3.6)."""
        x = images if isinstance(images, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(images)))
        if x.dtype != torch.uint8:
            raise TypeError(f"expected uint8 frames, got {x.dtype}")
        if x.dim() != 4 or x.shape[3] != 3:
            raise ValueError(f"expected (B,H,W,3) frames, got {tuple(x.shape)}")
        if not x.is_cuda:
            x = x.to(self.device)
        if max_det is None:
            max_det = self.face_detector.num_anchors(x.shape[1], x.shape[2])
        with torch.no_grad():
            dets, counts, _ = self.face_detector.detect_u8(x, max_det, reverse_channels=reverse_channels)
        counts = counts.cpu().numpy()
        dets = dets[:, :int(counts.max(initial=0))].cpu().numpy()   # only the rows that hold boxes cross to the host
        return [dets[i, :counts[i]].copy() for i in range(dets.shape[0])]
