"""`FaceAlignment` as inference.py uses it (face_detection/api.py:46-79 of the reference): a face detector behind
`get_detections_for_batch`.  Only the 'sfd' detector exists."""
from enum import Enum

import numpy as np


class LandmarksType(Enum):
    _2D = 1
    _2halfD = 2
    _3D = 3


class NetworkSize(Enum):
    LARGE = 4

    def __int__(self):
        return self.value


class FaceAlignment:
    def __init__(self, landmarks_type, network_size=NetworkSize.LARGE, device="cuda", flip_input=False, face_detector="sfd",
                 verbose=False, path_to_detector=None):
        if face_detector != "sfd":
            raise ValueError("only the S3FD ('sfd') detector is provided")
        from .detection.sfd import FaceDetector
        self.device, self.flip_input, self.landmarks_type, self.verbose = device, flip_input, landmarks_type, verbose
        self.face_detector = FaceDetector(device=device, verbose=verbose, path_to_detector=path_to_detector)

    def get_detections_for_batch(self, images):
        """images: (B,H,W,3) uint8, as inference.py passes them: cv2's BGR frames (inference.py:113 -> :78).  api.py:64
        reverses the channels before the detector, so the network sees them in RGB order.
        Returns, per image, the first surviving detection as (x1, y1, x2, y2) ints clipped at 0, or None."""
        bgr = np.ascontiguousarray(np.asarray(images)[..., ::-1])
        out = []
        for dets in self.face_detector.detect_from_batch(bgr):
            if len(dets) == 0:
                out.append(None)
                continue
            d = np.clip(dets[0], 0, None)
            out.append(tuple(int(v) for v in d[:4]))
        return out

    def get_detections_for_batch_u8(self, images):
        """`get_detections_for_batch` with the whole detector on the device (`w2l_s3fd_detect_u8`, one box per image):
        images (B,H,W,3) uint8 as for `get_detections_for_batch` (the channels are reversed on the device, as api.py:64
        does), a CUDA tensor or host memory.  Same result, up to exactly tied top scores."""
        out = []
        for dets in self.face_detector.detect_from_batch_u8(images, max_det=1, reverse_channels=True):
            if len(dets) == 0:
                out.append(None)
                continue
            d = np.clip(dets[0], 0, None)
            out.append(tuple(int(v) for v in d[:4]))
        return out


def face_boxes(rects, H, W, pads=(0, 10, 0, 0), nosmooth=False):
    """inference.py:87-103 on the detector's rectangles: pad (pads = top, bottom, left, right), clip to the H x W frame,
    smooth over a window of 5 frames unless nosmooth -> (F, 4) int64 rows (y1, y2, x1, x2), the crop rows of
    `Wav2Lip.infer_frames`.  Keeps the reference's arithmetic: the window mean is truncated into the integer array, the
    tail window `boxes[F-5:]` includes rows already smoothed, and with fewer than 5 frames its negative start counts from
    the end.  A frame without a face (None) raises ValueError naming the frame."""
    results = []
    pady1, pady2, padx1, padx2 = pads
    for i, rect in enumerate(rects):
        if rect is None:
            raise ValueError(f"Face not detected in frame {i}! Ensure the video contains a face in all the frames.")
        y1 = max(0, rect[1] - pady1)
        y2 = min(H, rect[3] + pady2)
        x1 = max(0, rect[0] - padx1)
        x2 = min(W, rect[2] + padx2)
        results.append([x1, y1, x2, y2])
    if not results:
        return np.zeros((0, 4), dtype=np.int64)
    boxes = np.array(results, dtype=np.int64)
    if not nosmooth:
        T = 5
        for i in range(len(boxes)):
            window = boxes[len(boxes) - T:] if i + T > len(boxes) else boxes[i: i + T]
            boxes[i] = np.mean(window, axis=0)
    return boxes[:, [1, 3, 0, 2]].copy()
