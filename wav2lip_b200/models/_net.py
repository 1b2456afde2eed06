"""Shared machinery of the three network mirrors: module tree from the C-side table, weight
hand-off to the context, and the no-fallback guards."""
import ctypes as C
import os

import torch
from torch import nn

from ._bridge import lib as _lib
from .conv import block_from_info


def build_tree(module: nn.Module, net: int):
    """Attach blocks under the reference's module paths, e.g. 'face_encoder_blocks.3.1' ->
    module.face_encoder_blocks[3][1] (ModuleList of Sequential), 'audio_encoder.7' ->
    module.audio_encoder[7] (Sequential)."""
    groups = {}
    for info in _lib.net_layers(net):
        parts = info["name"].split(".")
        groups.setdefault(parts[0], []).append((parts[1:], info))
    for top, rows in groups.items():
        if len(rows[0][0]) == 1:  # flat Sequential
            seq = nn.Sequential()
            for idx, info in rows:
                seq.add_module(idx[0], block_from_info(info))
            setattr(module, top, seq)
        else:  # ModuleList of Sequential
            stages = {}
            for idx, info in rows:
                stages.setdefault(int(idx[0]), nn.Sequential()).add_module(idx[1], block_from_info(info))
            setattr(module, top, nn.ModuleList([stages[i] for i in range(len(stages))]))


class NativeNet(nn.Module):
    NET = -1
    precision = _lib.PREC_F16

    def __init__(self):
        super().__init__()
        self._w2l_ctx = None
        self._w2l_key = None

    # --- context / weights -------------------------------------------------------------------
    def _device_index(self, ref: torch.Tensor) -> int:
        if not ref.is_cuda:
            raise _lib.W2LError(
                f"{type(self).__name__} runs on a CUDA (sm_90) device only; got a {ref.device} tensor. "
                "wav2lip_b200 has no CPU fallback.")
        return ref.device.index if ref.device.index is not None else torch.cuda.current_device()

    # --- change detection: cheap per call (the forward itself is ~2 ms at N=128) --------------------
    def _apply(self, fn, *args, **kwargs):  # .to() / .cuda() / .half() ... replace tensors
        out = super()._apply(fn, *args, **kwargs)
        self._w2l_tensors = None
        return out

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        self._w2l_tensors = None
        return out

    def mark_weights_dirty(self):
        """Call after mutating parameters behind autograd's back (e.g. through `.data`)."""
        self._w2l_tensors = None

    def _weights_key(self):
        ts = getattr(self, "_w2l_tensors", None)
        if ts is None:
            ts = [t for t in self.state_dict(keep_vars=True).values()]
            self._w2l_tensors = ts
            self._w2l_key = None
        return tuple(t._version for t in ts)

    def _ensure(self, ref: torch.Tensor):
        if self.training and self.NET != _lib.NET_DISC:
            # (the mirrors' forward() routes train mode to wav2lip_b200.training before it gets here)
            raise NotImplementedError(
                "this entry point runs the inference plan (BatchNorm on running statistics): call .eval(); the "
                "train-mode forward / backward is Module.forward() in train mode (wav2lip_b200/training.py)")
        dev = self._device_index(ref)
        if self._w2l_ctx is None or self._w2l_ctx.device != dev:
            self._w2l_ctx = _lib.Context(dev, self.precision)
            self._w2l_key = None
        key = self._weights_key()
        if key != self._w2l_key:
            stream = torch.cuda.current_stream(ref.device).cuda_stream
            self._load_into(self._w2l_ctx, stream)
            self._w2l_key = key
            self._w2l_range_checked = False
            if self.precision != _lib.PREC_BF16:
                # the flag is one per DEVICE (any context's kernels set it): start this model's check window clean
                self._w2l_ctx.f16_overflow(clear=True, stream=stream)
        return self._w2l_ctx

    def _load_into(self, ctx, stream):
        """Hand the current parameters to `ctx` (w2l_load_weights of this network)."""
        tensors, keep = {}, []
        for name, t in self.state_dict(keep_vars=True).items():
            if not t.dtype.is_floating_point:
                continue
            if not t.is_cuda:
                raise _lib.W2LError(f"parameter {name} is on {t.device}; move the module with .to('cuda') first")
            tc = t.detach().contiguous().float()
            keep.append(tc)
            tensors[name] = (tc.data_ptr(), tc.numel())
        ctx.load_weights(self.NET, tensors, stream)

    def _wants_grad(self) -> bool:
        return any(p.requires_grad for p in self.parameters())

    def _same_device(self, ctx, *tensors):
        """Every tensor whose data_ptr() crosses the C-ABI must live on the context's device: a CPU tensor or a tensor
        of another GPU would be dereferenced as a foreign pointer (illegal address -> sticky CUDA error).  The reference
        raises a device-mismatch RuntimeError in the same situation; so do we, before anything is launched."""
        for t in tensors:
            if t is None:
                continue
            idx = t.device.index if t.device.index is not None else (torch.cuda.current_device() if t.is_cuda else -1)
            if not t.is_cuda or idx != ctx.device:
                raise _lib.W2LError(
                    f"{type(self).__name__}: expected every input on cuda:{ctx.device}, got a tensor on {t.device} "
                    "(wav2lip_b200 has no CPU path and does not copy between devices)")

    def _range_guard(self, ctx, stream):
        """fp16 range guard (include/w2l.h: w2l_f16_overflow): checked once after the first forward that follows a
        weight (re)load — or after every forward with W2L_CHECK_RANGE=always — so a checkpoint whose activations leave
        the fp16 range raises instead of returning inf/NaN-poisoned results.  Costs one stream sync when it runs."""
        if self.precision == _lib.PREC_BF16:
            return
        if getattr(self, "_w2l_range_checked", False) and os.environ.get("W2L_CHECK_RANGE", "") != "always":
            return
        self._w2l_range_checked = True
        if ctx.f16_overflow(clear=True, stream=stream):
            raise _lib.W2LError(
                f"{type(self).__name__}: an activation left the fp16 range (|v| > 65504) with these weights/inputs; "
                "the result is not trustworthy. Run this checkpoint with bf16 operands: set "
                f"`{type(self).__name__}.precision = wav2lip_b200._lib.PREC_BF16` before the first forward.")

    @staticmethod
    def _in(t: torch.Tensor) -> torch.Tensor:
        return t.detach().contiguous().float()

    @staticmethod
    def _p(t: torch.Tensor):
        return C.c_void_p(t.data_ptr())

    def debug_layer_output(self, layer_index: int) -> torch.Tensor:
        """Output of block `layer_index` of the last forward as (N,C,H,W) fp32 (needs set_debug(True))."""
        ctx = self._w2l_ctx
        n, c, h, w = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _lib.check(ctx.lib.w2l_debug_layer_output(ctx.h, self.NET, layer_index, None, C.byref(n), C.byref(c),
                                                  C.byref(h), C.byref(w), None))
        y = torch.empty((n.value, c.value, h.value, w.value), device=f"cuda:{ctx.device}", dtype=torch.float32)
        stream = torch.cuda.current_stream(y.device).cuda_stream
        _lib.check(ctx.lib.w2l_debug_layer_output(ctx.h, self.NET, layer_index, self._p(y), None, None, None, None,
                                                  C.c_void_p(stream)))
        return y
