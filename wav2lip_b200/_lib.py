"""ctypes binding of libw2l.so — the declarations of include/w2l.h, nothing else.

The library is built in-tree by `python -c "import __graft_entry__ as g; g.build()"`
(nvcc -gencode arch=compute_90a,code=sm_90a).  If it is missing, importing this module still
works (so that error messages are useful) but any use raises W2LError: there is no fallback path.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))

W2L_OK, W2L_EINVAL, W2L_ENODEV, W2L_ECUDA, W2L_ENOMEM, W2L_ESTATE = 0, -1, -2, -3, -4, -5
NET_GENERATOR, NET_SYNCNET, NET_DISC, NET_S3FD = 0, 1, 2, 3
BLOCK_CONV_BN_RELU, BLOCK_CONVT_BN_RELU, BLOCK_CONV_LRELU, BLOCK_CONV_PLAIN, BLOCK_CONV_RELU = 0, 1, 2, 3, 4
PREC_F16, PREC_BF16, PREC_F32X = 0, 1, 2
TRAIN_WGRAD, TRAIN_ACCUMULATE, TRAIN_INPUT_GRAD, TRAIN_NO_STAT_UPDATE = 1, 2, 4, 8

# every symbol include/w2l.h declares (tests/test_abi.py checks the header against this list)
EXPORTS = [
    "w2l_abi_version", "w2l_last_error", "w2l_net_num_layers", "w2l_net_layer_info",
    "w2l_create", "w2l_destroy", "w2l_load_weights",
    "w2l_generator_forward", "w2l_generator_forward_host", "w2l_generator_forward_u8", "w2l_generator_forward_u8_host",
    "w2l_generator_submit_host", "w2l_generator_submit_u8_host", "w2l_host_wait",
    "w2l_syncnet_forward", "w2l_syncnet_forward_frames", "w2l_cosine_bce_loss", "w2l_l1_loss", "w2l_disc_forward",
    "w2l_conv_block_forward", "w2l_debug_layer_output",
    "w2l_melspectrogram", "w2l_melspectrogram_host", "w2l_mel_num_frames", "w2l_mel_num_chunks", "w2l_mel_chunks",
    "w2l_set_debug", "w2l_mel_basis_host", "w2l_launch_count", "w2l_device_bytes", "w2l_profile_plan",
    "w2l_f16_overflow",
    "w2l_crop_resize_u8", "w2l_paste_u8", "w2l_lipsync_frames_u8", "w2l_s3fd_out_dims", "w2l_s3fd_forward",
    "w2l_train_bind", "w2l_train_forward", "w2l_train_backward", "w2l_adam_step", "w2l_wav2lip_train_step",
    "w2l_hq_wav2lip_train_step", "w2l_syncnet_train_step", "w2l_adam_state",
    "w2l_train_last_output", "w2l_train_flops", "w2l_comm_unique_id", "w2l_comm_init", "w2l_conv_block_train", "w2l_train_profile",
    "w2l_debug_kernel_table", "w2l_debug_plan_kernels", "w2l_debug_set_sm_count", "w2l_debug_train_blocks", "w2l_debug_train_tensor",
    "w2l_s3fd_detect_u8", "w2l_debug_s3fd_candidates", "w2l_face_crops_u8", "w2l_train_batch_wav2lip", "w2l_train_batch_syncnet",
    "w2l_resample_num_samples", "w2l_resample", "w2l_resample_filter_host", "w2l_resample_final",
    "w2l_melstream_create", "w2l_melstream_pending", "w2l_melstream_push", "w2l_melstream_finish", "w2l_melstream_destroy",
    "w2l_melstream_set_input_rate", "w2l_stream_set_input_rate", "w2l_stream_group_set_input_rate",
    "w2l_stream_schedule", "w2l_stream_create", "w2l_stream_pending", "w2l_stream_push", "w2l_stream_finish",
    "w2l_stream_destroy", "w2l_stream_detect_need",
    "w2l_stream_group_create", "w2l_stream_group_open", "w2l_stream_group_open_detect", "w2l_stream_group_close",
    "w2l_stream_group_pending",
    "w2l_stream_group_tick", "w2l_stream_group_error", "w2l_stream_group_buckets", "w2l_stream_group_counters",
    "w2l_stream_group_destroy",
]
STREAM_ROW = 7  # W2L_STREAM_ROW: output index, chunk start, frame index, y1, y2, x1, x2
KFAM_IGEMM, KFAM_PATCH, KFAM_CONVT_FUSED = 0, 1, 2
WG_PLAIN, WG_STRIDED, WG_TRANSPOSED, WG_SWAP, WG_FOLDED = 0, 1, 2, 3, 4
TAPE_X, TAPE_Z, TAPE_Y, TAPE_DY, TAPE_DZ, TAPE_DU, TAPE_DX, TAPE_DX_ADD, TAPE_STATS, TAPE_F32 = range(10)


class W2LError(RuntimeError):
    pass


class StreamDesc(C.Structure):
    """w2l_stream_desc (include/w2l.h)."""
    _fields_ = [("F", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("fps", C.c_double), ("nosmooth", C.c_int32),
                ("has_box", C.c_int32), ("box", C.c_int32 * 4), ("pads", C.c_int32 * 4)]


class LayerInfo(C.Structure):
    _fields_ = [("name", C.c_char * 64), ("kind", C.c_int32), ("cin", C.c_int32), ("cout", C.c_int32),
                ("kh", C.c_int32), ("kw", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
                ("ph", C.c_int32), ("pw", C.c_int32), ("out_pad", C.c_int32), ("residual", C.c_int32), ("cout_real", C.c_int32)]


class KernelInfo(C.Structure):
    _fields_ = [("name", C.c_char * 64), ("family", C.c_int32), ("bn", C.c_int32), ("bk", C.c_int32), ("mt", C.c_int32),
                ("head", C.c_int32), ("bf16", C.c_int32), ("x2", C.c_int32), ("tma_epi", C.c_int32), ("fold", C.c_int32),
                ("m_tiles", C.c_int32), ("n_tiles", C.c_int32), ("grid", C.c_int32),
                ("box_w", C.c_int32), ("box_h", C.c_int32), ("box_n", C.c_int32), ("patch_th", C.c_int32)]

    def as_dict(self) -> dict:
        d = {f: getattr(self, f) for f, _ in self._fields_}
        d["name"] = self.name.decode()
        return d


class TrainBlockInfo(C.Structure):
    _fields_ = ([("name", C.c_char * 64)]
                + [(f, C.c_int32) for f in (
                    "layer", "kind", "cin", "cout", "kh", "kw", "sh", "sw", "ph", "pw", "out_pad", "residual",
                    "n", "h_in", "w_in", "h_out", "w_out", "lane", "has_dx", "has_dx_add", "has_du", "has_wgrad",
                    "wg_bn", "wg_form", "wg_ntaps", "wg_tg", "wg_ngroups", "wg_p", "wg_bw", "wg_bh", "wg_bnb",
                    "wg_chunks", "wg_m_tiles", "wg_n_tiles", "wg_splits", "wg_grid", "n_fwd", "n_dgrad")]
                + [("fwd", KernelInfo * 4), ("dgrad", KernelInfo * 4)])

    def as_dict(self) -> dict:
        d = {f: getattr(self, f) for f, _ in self._fields_ if f not in ("name", "fwd", "dgrad")}
        d["name"] = self.name.decode()
        d["fwd"] = [self.fwd[i].as_dict() for i in range(self.n_fwd)]
        d["dgrad"] = [self.dgrad[i].as_dict() for i in range(self.n_dgrad)]
        return d


def _kernel_rows(fn) -> list:
    n = fn(0, None)
    if n < 0:
        check(n)
    buf = (KernelInfo * max(n, 1))()
    k = fn(n, buf)
    if k < 0:
        check(k)
    return [buf[i].as_dict() for i in range(k)]


def kernel_table() -> list:
    """Every compiled conv kernel instantiation as a list of dicts (host only, no GPU needed)."""
    lib = get_lib()
    return _kernel_rows(lambda cap, out: lib.w2l_debug_kernel_table(cap, out))


def lib_path() -> str:
    return os.environ.get("W2L_LIB", os.path.join(HERE, "libw2l.so"))


_lib: Optional[C.CDLL] = None


def get_lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise W2LError(
            f"{path} not found: build it with `python -c \"import __graft_entry__ as g; g.build()\"`. "
            "wav2lip_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(path)
    vp, i32, i64, cp = C.c_void_p, C.c_int, C.c_int64, C.c_char_p
    lib.w2l_abi_version.restype = i32
    lib.w2l_last_error.restype = cp
    lib.w2l_net_num_layers.argtypes = [i32]
    lib.w2l_net_layer_info.argtypes = [i32, i32, C.POINTER(LayerInfo)]
    lib.w2l_create.argtypes = [i32, i32, C.POINTER(vp)]
    lib.w2l_destroy.argtypes = [vp]
    lib.w2l_set_debug.argtypes = [vp, i32]
    lib.w2l_load_weights.argtypes = [vp, i32, i32, C.POINTER(cp), C.POINTER(vp), C.POINTER(i64), vp]
    lib.w2l_generator_forward.argtypes = [vp, vp, vp, vp, i32, i32, vp]
    lib.w2l_generator_forward_host.argtypes = [vp, vp, vp, vp, i32, i32]
    lib.w2l_generator_forward_u8.argtypes = [vp, vp, vp, vp, i32, vp]
    lib.w2l_generator_forward_u8_host.argtypes = [vp, vp, vp, vp, i32]
    lib.w2l_generator_submit_host.argtypes = [vp, vp, vp, vp, i32, i32]
    lib.w2l_generator_submit_u8_host.argtypes = [vp, vp, vp, vp, i32]
    lib.w2l_host_wait.argtypes = [vp, i32]
    lib.w2l_mel_num_chunks.argtypes = [i64, C.c_double]
    lib.w2l_mel_num_chunks.restype = i64
    lib.w2l_mel_chunks.argtypes = [vp, vp, i64, C.c_double, vp, i64, vp]
    lib.w2l_syncnet_forward.argtypes = [vp, vp, vp, vp, vp, i32, vp]
    lib.w2l_disc_forward.argtypes = [vp, vp, vp, i32, i32, vp]
    lib.w2l_syncnet_forward_frames.argtypes = [vp, vp, vp, vp, vp, i32, i32, vp]
    lib.w2l_cosine_bce_loss.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.w2l_l1_loss.argtypes = [vp, vp, vp, i64, vp, vp]
    lib.w2l_conv_block_forward.argtypes = [vp, C.POINTER(LayerInfo), vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.w2l_debug_layer_output.argtypes = [vp, i32, i32, vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), vp]
    lib.w2l_melspectrogram.argtypes = [vp, vp, i64, vp, vp]
    lib.w2l_melspectrogram_host.argtypes = [vp, vp, i64, vp]
    lib.w2l_mel_num_frames.argtypes = [i64]
    lib.w2l_mel_num_frames.restype = i64
    lib.w2l_mel_basis_host.argtypes = [vp]
    lib.w2l_launch_count.argtypes = [vp]
    lib.w2l_launch_count.restype = i64
    lib.w2l_device_bytes.argtypes = [vp]
    lib.w2l_device_bytes.restype = i64
    lib.w2l_profile_plan.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp]
    lib.w2l_f16_overflow.argtypes = [vp, i32, C.POINTER(i32), vp]
    f32 = C.c_float
    lib.w2l_s3fd_out_dims.argtypes = [i32, i32, C.POINTER(i32)]
    lib.w2l_s3fd_forward.argtypes = [vp, vp, C.POINTER(vp), i32, i32, i32, vp]
    lib.w2l_s3fd_detect_u8.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp, C.POINTER(vp), vp]
    lib.w2l_debug_s3fd_candidates.argtypes = [vp, i32, i32, vp, C.POINTER(i32), C.POINTER(i32)]
    lib.w2l_face_crops_u8.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32, i32, i32, vp, vp, vp, i64, vp]
    lib.w2l_crop_resize_u8.argtypes = [vp, vp, i32, i32, i32, C.POINTER(i32), i32, vp, vp]
    lib.w2l_paste_u8.argtypes = [vp, vp, vp, i32, i32, i32, C.POINTER(i32), i32, vp, vp]
    lib.w2l_lipsync_frames_u8.argtypes = [vp, vp, vp, i32, i32, i32, C.POINTER(i32), i32, vp, vp]
    lib.w2l_train_batch_wav2lip.argtypes = [vp, vp, i64, vp, i64, vp, i32, vp, vp, vp, vp, vp]
    lib.w2l_train_batch_syncnet.argtypes = [vp, vp, i64, vp, i64, vp, i32, vp, vp, vp, vp]
    lib.w2l_train_bind.argtypes = [vp, i32, i32, C.POINTER(cp), C.POINTER(vp), C.POINTER(vp), C.POINTER(i64)]
    lib.w2l_train_forward.argtypes = [vp, i32, vp, vp, vp, vp, i32, i32, i32, vp]
    lib.w2l_train_backward.argtypes = [vp, i32, vp, vp, vp, i32, vp]
    lib.w2l_adam_step.argtypes = [vp, i32, f32, f32, f32, f32, vp]
    lib.w2l_wav2lip_train_step.argtypes = [vp, vp, vp, vp, vp, i32, i32, f32, f32, vp, vp]
    lib.w2l_train_last_output.argtypes = [vp, vp, i64, vp]
    lib.w2l_hq_wav2lip_train_step.argtypes = [vp, vp, vp, vp, vp, i32, i32, f32, f32, f32, f32, vp, vp]
    lib.w2l_syncnet_train_step.argtypes = [vp, vp, vp, vp, i32, f32, vp, vp]
    lib.w2l_adam_state.argtypes = [vp, i32, i32, i32, C.POINTER(cp), C.POINTER(vp), C.POINTER(vp), C.POINTER(i64), vp]
    lib.w2l_train_flops.argtypes = [vp, i32]
    lib.w2l_train_flops.restype = C.c_double
    lib.w2l_train_profile.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp]
    lib.w2l_comm_unique_id.argtypes = [vp, C.c_char_p]
    lib.w2l_comm_init.argtypes = [vp, C.c_char_p, i32, i32]
    lib.w2l_conv_block_train.argtypes = [vp, C.POINTER(LayerInfo), vp, i32, i32, i32] + [vp] * 14
    lib.w2l_debug_kernel_table.argtypes = [i32, C.POINTER(KernelInfo)]
    lib.w2l_debug_plan_kernels.argtypes = [vp, i32, i32, C.POINTER(KernelInfo)]
    lib.w2l_debug_set_sm_count.argtypes = [vp, i32]
    lib.w2l_debug_train_blocks.argtypes = [vp, i32, i32, C.POINTER(TrainBlockInfo)]
    lib.w2l_debug_train_tensor.argtypes = [vp, i32, i32, i32, vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32),
                                           C.POINTER(i32), vp]
    pi64 = C.POINTER(i64)
    lib.w2l_melstream_create.argtypes = [vp, i32, C.POINTER(vp)]
    lib.w2l_melstream_pending.argtypes = [vp, i64, i32]
    lib.w2l_melstream_pending.restype = i64
    lib.w2l_melstream_push.argtypes = [vp, vp, i64, vp, i64, pi64, C.POINTER(i32), vp]
    lib.w2l_melstream_finish.argtypes = [vp, vp, i64, pi64, C.POINTER(i32), vp]
    lib.w2l_melstream_destroy.argtypes = [vp]
    lib.w2l_resample_num_samples.argtypes = [i32, i32, i64]
    lib.w2l_resample_num_samples.restype = i64
    lib.w2l_resample.argtypes = [vp, vp, i64, i32, i32, vp, i64, vp]
    lib.w2l_resample_filter_host.argtypes = [vp]
    lib.w2l_resample_final.argtypes = [i32, i64, i32, pi64]
    lib.w2l_melstream_set_input_rate.argtypes = [vp, i32]
    lib.w2l_stream_set_input_rate.argtypes = [vp, i32]
    lib.w2l_stream_group_set_input_rate.argtypes = [vp, i32, i32]
    lib.w2l_stream_schedule.argtypes = [C.POINTER(StreamDesc), vp, i64, i32, i64, i64, vp, pi64]
    lib.w2l_stream_detect_need.argtypes = [C.POINTER(StreamDesc), i64, i32, pi64]
    lib.w2l_stream_create.argtypes = [vp, vp, C.POINTER(StreamDesc), vp, i32, C.POINTER(vp)]
    lib.w2l_stream_pending.argtypes = [vp, i64, i32, pi64]
    lib.w2l_stream_push.argtypes = [vp, vp, i64, vp, i64, pi64, pi64, vp]
    lib.w2l_stream_finish.argtypes = [vp, vp, i64, pi64, pi64, vp]
    lib.w2l_stream_destroy.argtypes = [vp]
    lib.w2l_stream_group_create.argtypes = [vp, i32, i32, C.POINTER(vp)]
    lib.w2l_stream_group_open.argtypes = [vp, vp, C.POINTER(StreamDesc), vp, C.POINTER(i32)]
    lib.w2l_stream_group_open_detect.argtypes = [vp, vp, C.POINTER(StreamDesc), C.POINTER(i32)]
    lib.w2l_stream_group_close.argtypes = [vp, i32]
    lib.w2l_stream_group_pending.argtypes = [vp, i32, vp, vp, vp, vp]
    lib.w2l_stream_group_tick.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.w2l_stream_group_error.argtypes = [vp, i32]
    lib.w2l_stream_group_error.restype = cp
    lib.w2l_stream_group_buckets.argtypes = [i32, i64, vp, i64]
    lib.w2l_stream_group_counters.argtypes = [vp, pi64, pi64, pi64]
    lib.w2l_stream_group_destroy.argtypes = [vp]
    for name in EXPORTS:
        getattr(lib, name)  # AttributeError here == header / library mismatch
    if lib.w2l_abi_version() != 1:
        raise W2LError(f"ABI version mismatch: library {lib.w2l_abi_version()}, binding 1")
    _lib = lib
    return lib


def check(code: int) -> None:
    if code != W2L_OK:
        msg = get_lib().w2l_last_error().decode("utf-8", "replace")
        raise W2LError(f"libw2l error {code}: {msg}")


def net_layers(net: int):
    """The architecture table of `net` as a list of dicts (host only, no GPU needed)."""
    lib = get_lib()
    n = lib.w2l_net_num_layers(net)
    if n < 0:
        check(n)
    out = []
    for i in range(n):
        li = LayerInfo()
        check(lib.w2l_net_layer_info(net, i, C.byref(li)))
        out.append({"name": li.name.decode(), "kind": li.kind, "cin": li.cin, "cout": li.cout,
                    "k": (li.kh, li.kw), "stride": (li.sh, li.sw), "pad": (li.ph, li.pw),
                    "out_pad": li.out_pad, "residual": bool(li.residual), "cout_real": li.cout_real})
    return out


class Context:
    """Owns one w2l_ctx (one device, one precision).  Not thread safe."""

    def __init__(self, device: int = 0, precision: int = PREC_F16):
        self.lib = get_lib()
        h = C.c_void_p()
        check(self.lib.w2l_create(int(device), int(precision), C.byref(h)))
        self.h = h
        self.device = int(device)

    def close(self):
        if getattr(self, "h", None):
            self.lib.w2l_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def launch_count(self) -> int:
        return int(self.lib.w2l_launch_count(self.h))

    def device_bytes(self) -> int:
        return int(self.lib.w2l_device_bytes(self.h))

    def f16_overflow(self, clear: bool = True, stream: int = 0) -> bool:
        """True if an fp16 epilogue stored an inf/NaN activation since the flag was last cleared (synchronises)."""
        flag = C.c_int(0)
        check(self.lib.w2l_f16_overflow(self.h, 1 if clear else 0, C.byref(flag), C.c_void_p(stream)))
        return bool(flag.value)

    def set_debug(self, keep_all: bool):
        check(self.lib.w2l_set_debug(self.h, 1 if keep_all else 0))

    def plan_kernels(self, net: int) -> list:
        """The conv launches of the last plan of `net` (-1: of the last w2l_conv_block_forward) as a list of dicts."""
        return _kernel_rows(lambda cap, out: self.lib.w2l_debug_plan_kernels(self.h, int(net), cap, out))

    def set_sm_count(self, n: int):
        """Build later inference plans for n SMs (1 .. the device's count; 0 restores it); drops the cached plans."""
        check(self.lib.w2l_debug_set_sm_count(self.h, int(n)))

    def train_blocks(self, net: int) -> list:
        """The blocks of the last training plan of `net` (-1: of the last w2l_conv_block_train) as a list of dicts."""
        n = self.lib.w2l_debug_train_blocks(self.h, int(net), 0, None)
        if n < 0:
            check(n)
        buf = (TrainBlockInfo * max(n, 1))()
        k = self.lib.w2l_debug_train_blocks(self.h, int(net), n, buf)
        if k < 0:
            check(k)
        return [buf[i].as_dict() for i in range(k)]

    def train_tensor(self, net: int, block: int, which: int, stream: int = 0):
        """One tape tensor of a block of the last training plan of `net` (TAPE_*) as a float32 CUDA tensor (NCHW; STATS:
        (2, C, 1, 1) = mean, invstd; F32: the fp32 output of SyncNet's last blocks, (N, C, 1, 1)), or None if the block
        has no such tensor.  Synchronises `stream`."""
        import torch
        d = [C.c_int32() for _ in range(4)]
        r = self.lib.w2l_debug_train_tensor(self.h, int(net), int(block), int(which), None, *[C.byref(v) for v in d], None)
        if r == W2L_EINVAL:
            return None
        check(r)
        out = torch.empty(tuple(v.value for v in d), device=f"cuda:{self.device}", dtype=torch.float32)
        check(self.lib.w2l_debug_train_tensor(self.h, int(net), int(block), int(which), C.c_void_p(out.data_ptr()),
                                              None, None, None, None, C.c_void_p(stream)))
        torch.cuda.synchronize(self.device)
        return out

    def s3fd_candidates(self, image: int, cap: int = None):
        """The sorted pre-NMS candidates (score > 0.5) of one image of the last S3FD detection as a float32 (n, 6) array
        (x1, y1, x2, y2, score, location index), and which NMS path ran (0: shared memory, 1: global).  Synchronises."""
        import numpy as np
        n, path = C.c_int32(), C.c_int32()
        check(self.lib.w2l_debug_s3fd_candidates(self.h, int(image), 0, None, C.byref(n), C.byref(path)))
        k = n.value if cap is None else min(int(cap), n.value)
        out = np.zeros((max(k, 1), 6), dtype=np.float32)
        check(self.lib.w2l_debug_s3fd_candidates(self.h, int(image), k, C.c_void_p(out.ctypes.data), C.byref(n),
                                                 C.byref(path)))
        return out[:k], int(path.value)

    def load_weights(self, net: int, tensors: dict, stream: int = 0):
        """tensors: name -> (device_ptr, numel) of fp32 contiguous CUDA tensors."""
        names = list(tensors.keys())
        n = len(names)
        arr_n = (C.c_char_p * n)(*[s.encode() for s in names])
        arr_p = (C.c_void_p * n)(*[tensors[s][0] for s in names])
        arr_c = (C.c_int64 * n)(*[tensors[s][1] for s in names])
        check(self.lib.w2l_load_weights(self.h, net, n, arr_n, arr_p, arr_c, C.c_void_p(stream)))

    def train_profile(self, net: int, iters: int = 3, stream: int = 0, cap: int = 512):
        ms = (C.c_float * cap)()
        fl = (C.c_double * cap)()
        names = ((C.c_char * 64) * cap)()
        k = self.lib.w2l_train_profile(self.h, net, iters, cap, ms, fl, names, C.c_void_p(stream))
        if k < 0:
            check(k)
        return [(names[i].value.decode(), float(ms[i]), float(fl[i])) for i in range(k)]

    def profile_plan(self, net: int, iters: int = 5, stream: int = 0, cap: int = 256):
        ms = (C.c_float * cap)()
        fl = (C.c_double * cap)()
        names = ((C.c_char * 64) * cap)()
        k = self.lib.w2l_profile_plan(self.h, net, iters, cap, ms, fl, names, C.c_void_p(stream))
        if k < 0:
            check(k)
        return [(names[i].value.decode(), float(ms[i]), float(fl[i])) for i in range(k)]
