"""Mirror of the reference's `face_detection` package surface that inference.py uses (inference.py:4, :75-100):
`face_detection.FaceAlignment(face_detection.LandmarksType._2D, flip_input=False, device=device)` and
`.get_detections_for_batch(images)`.  The S3FD network (face_detection/detection/sfd/net_s3fd.py:22-129) runs on the H100
core (`w2l_s3fd_forward`); the landmark networks of the reference package (FAN / ResNetDepth) are not used by Wav2Lip and
are not provided."""
from .api import FaceAlignment, LandmarksType, NetworkSize, face_boxes  # noqa: F401

__version__ = "1.0.1"
