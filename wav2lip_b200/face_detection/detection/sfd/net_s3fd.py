"""Mirror of the reference's `s3fd` module (face_detection/detection/sfd/net_s3fd.py:22-129): same attribute names and
state_dict keys (`conv1_1.weight` ... `conv7_2_mbox_loc.bias`, `conv3_3_norm.weight`), so the published s3fd.pth loads with
strict=True; `forward` is ONE call into libw2l.so (`w2l_s3fd_forward`) and returns the module's 12 maps."""
import ctypes as C
import importlib

import torch
from torch import nn

_lib = importlib.import_module(__name__.split(".face_detection")[0] + "._lib") if ".face_detection" in __name__ else None
if _lib is None:   # imported as the top-level package `face_detection` (wav2lip_b200/ on sys.path shadows the reference's)
    import os
    import sys
    _root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))))
    if _root not in sys.path:
        sys.path.append(_root)
    _lib = importlib.import_module("wav2lip_b200._lib")
_NativeNet = importlib.import_module("wav2lip_b200.models._net").NativeNet


class L2Norm(nn.Module):
    """Parameter holder of net_s3fd.py:6-19 (the normalisation itself is a kernel of the plan)."""

    def __init__(self, n_channels, scale=1.0):
        super().__init__()
        self.n_channels, self.scale, self.eps = n_channels, scale, 1e-10
        self.weight = nn.Parameter(torch.full((n_channels,), float(scale)))


class s3fd(_NativeNet):
    NET = _lib.NET_S3FD

    def __init__(self):
        super().__init__()
        layers = _lib.net_layers(self.NET)           # conv1_1 ... conv7_2 (19) and the twelve mbox heads, from the C-side table

        def add(info):
            cout = info["cout_real"] or info["cout"]
            setattr(self, info["name"], nn.Conv2d(info["cin"], cout, info["k"], info["stride"], info["pad"]))
        for info in layers[:19]:
            add(info)
        self.conv3_3_norm = L2Norm(256, scale=10)    # (registration order = the reference's state_dict order, net_s3fd.py:25-69)
        self.conv4_3_norm = L2Norm(512, scale=8)
        self.conv5_3_norm = L2Norm(512, scale=5)
        for info in layers[19:]:
            add(info)

    def forward(self, x):
        ctx = self._ensure(x)
        self._same_device(ctx, x)
        img = self._in(x)
        if img.dim() != 4 or img.shape[1] != 3 or img.shape[2] < 32 or img.shape[3] < 32:
            raise ValueError(f"expected (B,3,H,W) with H, W >= 32, got {tuple(img.shape)}")
        B, _, H, W = img.shape
        dims = (C.c_int32 * 12)()
        _lib.check(ctx.lib.w2l_s3fd_out_dims(H, W, dims))
        outs = []
        for i in range(6):
            outs.append(torch.empty((B, 2, dims[2 * i], dims[2 * i + 1]), device=img.device, dtype=torch.float32))
            outs.append(torch.empty((B, 4, dims[2 * i], dims[2 * i + 1]), device=img.device, dtype=torch.float32))
        if B == 0:
            return outs
        ptrs = (C.c_void_p * 12)(*[o.data_ptr() for o in outs])
        stream = torch.cuda.current_stream(img.device).cuda_stream
        _lib.check(ctx.lib.w2l_s3fd_forward(ctx.h, self._p(img), ptrs, B, H, W, C.c_void_p(stream)))
        self._range_guard(ctx, stream)
        return outs

    @staticmethod
    def num_anchors(H: int, W: int) -> int:
        """Locations of the six maps of an H x W image (the most boxes a detection can keep)."""
        dims = (C.c_int32 * 12)()
        _lib.check(_lib.get_lib().w2l_s3fd_out_dims(int(H), int(W), dims))
        return sum(dims[2 * i] * dims[2 * i + 1] for i in range(6))

    def detect_u8(self, frames: torch.Tensor, max_det: int, reverse_channels: bool = False, return_maps: bool = False):
        """The detector on the device (`w2l_s3fd_detect_u8`): frames (B,H,W,3) uint8 CUDA tensor in the order
        `detect_from_batch` takes them (reverse_channels: reversed first, as api.py:64 does) -> dets (B,max_det,5) float32
        (x1, y1, x2, y2, score; the first counts[b] rows are image b's boxes, best first, the rest zero), counts (B,)
        int32, and with return_maps the 12 maps `forward` returns for the same frames."""
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise TypeError(f"expected a uint8 torch tensor, got {getattr(frames, 'dtype', type(frames))}")
        if frames.dim() != 4 or frames.shape[3] != 3 or frames.shape[1] < 32 or frames.shape[2] < 32:
            raise ValueError(f"expected (B,H,W,3) with H, W >= 32, got {tuple(frames.shape)}")
        if isinstance(max_det, bool) or not isinstance(max_det, int) or max_det < 1:
            raise ValueError(f"max_det must be an int >= 1, got {max_det!r}")
        ctx = self._ensure(frames)
        self._same_device(ctx, frames)
        frames = frames.contiguous()
        B, H, W, _ = frames.shape
        dets = torch.empty((B, max_det, 5), device=frames.device, dtype=torch.float32)   # the NMS kernel zero-fills the tail
        counts = torch.zeros((B,), device=frames.device, dtype=torch.int32)
        outs, ptrs = None, None
        if return_maps:
            dims = (C.c_int32 * 12)()
            _lib.check(ctx.lib.w2l_s3fd_out_dims(H, W, dims))
            outs = []
            for i in range(6):
                for c in (2, 4):
                    outs.append(torch.empty((B, c, dims[2 * i], dims[2 * i + 1]), device=frames.device, dtype=torch.float32))
            ptrs = (C.c_void_p * 12)(*[o.data_ptr() for o in outs])
        if B == 0:
            return dets, counts, outs
        stream = torch.cuda.current_stream(frames.device).cuda_stream
        _lib.check(ctx.lib.w2l_s3fd_detect_u8(ctx.h, self._p(frames), B, H, W, 1 if reverse_channels else 0, max_det,
                                              self._p(dets), self._p(counts), ptrs, C.c_void_p(stream)))
        self._range_guard(ctx, stream)
        return dets, counts, outs
