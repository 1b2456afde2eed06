"""Parameter containers with the reference's block names and state_dict layout.

Mirrors /root/reference/models/conv.py: `Conv2d` (:5-19), `nonorm_Conv2d` (:21-31) and
`Conv2dTranspose` (:33-44) keep `conv_block = Sequential(conv[, BatchNorm2d])`, so the keys are
`<block>.conv_block.0.weight`, `<block>.conv_block.1.running_mean`, ... exactly as in released
checkpoints.  The torch.nn layers are used as parameter holders (and for their default init) only:
`forward` goes through the C-ABI operator `w2l_conv_block_forward`, never through torch's conv.
"""
import ctypes as C

import torch
from torch import nn

from ._bridge import lib as _lib


def _pair(v):
    return (v, v) if isinstance(v, int) else (int(v[0]), int(v[1]))


_ctx_cache = {}


def _shared_ctx(device_index: int):
    key = int(device_index)
    if key not in _ctx_cache:
        _ctx_cache[key] = _lib.Context(key)
    return _ctx_cache[key]


class _Block(nn.Module):
    KIND = _lib.BLOCK_CONV_BN_RELU

    def _spec(self):
        conv = self.conv_block[0]
        li = _lib.LayerInfo()
        li.name = b"block"
        li.kind = self.KIND
        li.cin, li.cout = conv.in_channels, conv.out_channels
        li.kh, li.kw = conv.kernel_size
        li.sh, li.sw = conv.stride
        li.ph, li.pw = conv.padding
        li.out_pad = conv.output_padding[0] if hasattr(conv, "output_padding") and self.KIND == _lib.BLOCK_CONVT_BN_RELU else 0
        li.residual = 1 if getattr(self, "residual", False) else 0
        return li

    def forward(self, x):
        if self.training and len(self.conv_block) > 1:
            raise NotImplementedError("training-mode BatchNorm (batch statistics) is not built yet: call .eval()")
        if not x.is_cuda:
            raise _lib.W2LError("wav2lip_b200 blocks run on a CUDA (sm_90) device only; there is no CPU path")
        x = x.contiguous().float()
        conv = self.conv_block[0]
        bn = self.conv_block[1] if len(self.conv_block) > 1 else None
        li = self._spec()
        n, _, h, w = x.shape
        if self.KIND == _lib.BLOCK_CONVT_BN_RELU:
            ho = (h - 1) * li.sh - 2 * li.ph + li.kh + li.out_pad
            wo = (w - 1) * li.sw - 2 * li.pw + li.kw + li.out_pad
        else:
            ho = (h + 2 * li.ph - li.kh) // li.sh + 1
            wo = (w + 2 * li.pw - li.kw) // li.sw + 1
        y = torch.empty((n, li.cout, ho, wo), device=x.device, dtype=torch.float32)
        ctx = _shared_ctx(x.device.index or 0)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
        f = lambda t: t.detach().contiguous().float() if t is not None else None
        wt, b = f(conv.weight), f(conv.bias)
        g, be, m, v = (f(bn.weight), f(bn.bias), f(bn.running_mean), f(bn.running_var)) if bn is not None else (None,) * 4
        stream = torch.cuda.current_stream(x.device).cuda_stream
        _lib.check(ctx.lib.w2l_conv_block_forward(ctx.h, C.byref(li), ptr(x), n, h, w, ptr(wt), ptr(b), ptr(g), ptr(be),
                                                  ptr(m), ptr(v), ptr(y), C.c_void_p(stream)))
        return y


class Conv2d(_Block):
    KIND = _lib.BLOCK_CONV_BN_RELU

    def __init__(self, cin, cout, kernel_size, stride, padding, residual=False, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_block = nn.Sequential(nn.Conv2d(cin, cout, kernel_size, stride, padding), nn.BatchNorm2d(cout))
        self.residual = residual


class nonorm_Conv2d(_Block):
    KIND = _lib.BLOCK_CONV_LRELU

    def __init__(self, cin, cout, kernel_size, stride, padding, residual=False, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_block = nn.Sequential(nn.Conv2d(cin, cout, kernel_size, stride, padding))
        # conv.py:22-31 accepts `residual` and ignores it


class Conv2dTranspose(_Block):
    KIND = _lib.BLOCK_CONVT_BN_RELU

    def __init__(self, cin, cout, kernel_size, stride, padding, output_padding=0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_block = nn.Sequential(nn.ConvTranspose2d(cin, cout, kernel_size, stride, padding, output_padding),
                                        nn.BatchNorm2d(cout))


def block_from_info(info):
    """Build the container for one row of a C-side architecture table (w2l_net_layer_info)."""
    k, s, p = info["k"], info["stride"], info["pad"]
    if info["kind"] == _lib.BLOCK_CONV_BN_RELU:
        return Conv2d(info["cin"], info["cout"], k, s, p, residual=info["residual"])
    if info["kind"] == _lib.BLOCK_CONVT_BN_RELU:
        return Conv2dTranspose(info["cin"], info["cout"], k, s, p, info["out_pad"])
    if info["kind"] == _lib.BLOCK_CONV_LRELU:
        return nonorm_Conv2d(info["cin"], info["cout"], k, s, p)
    raise ValueError(info)
