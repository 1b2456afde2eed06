"""Every kernel variant of the conv path gives the same network output: the specialised kernels (patch kernel
with resident weights, K-folded first layers, two M tiles per CTA, fused 4-phase transposed conv) can be switched
off one by one through W2L_DISABLE_* (read when a context is created), falling back to the generic
implicit-GEMM kernel.  Also: the host-buffer entry point (chunked, 3-stream pipelined) is bit-identical to the
device-resident call."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import w2l_oracle as O

pytestmark = pytest.mark.gpu

FLAGS = ["W2L_DISABLE_HALO", "W2L_DISABLE_FOLD", "W2L_DISABLE_CTFUSED", "W2L_DISABLE_MT2", "W2L_DISABLE_TMAEPI", "W2L_DISABLE_FOLDS2",
         "W2L_DISABLE_SIDESTREAM"]


def _fresh_generator(env):
    from wav2lip_b200.models import Wav2Lip
    keys = FLAGS
    old = {k: os.environ.get(k) for k in keys}
    try:
        for k in keys:
            os.environ.pop(k, None)
        os.environ.update(env)
        g = Wav2Lip()
        g.load_state_dict(O.make_state_dict("generator", 0), strict=True)
        g = g.cuda().eval()
        with torch.no_grad():
            g._ensure(torch.zeros(1, device="cuda"))  # the context (and its flags) is created here
        return g
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.parametrize("env", [{}, {"W2L_DISABLE_HALO": "1"}, {"W2L_DISABLE_FOLD": "1"},
                                 {"W2L_DISABLE_CTFUSED": "1"}, {"W2L_DISABLE_MT2": "1"}, {k: "1" for k in FLAGS}],
                         ids=["all-on", "no-patch", "no-fold", "no-fused-convT", "no-mt2", "generic-only"])
def test_generator_variants_agree_with_oracle(env, golden_dir):
    gold = np.load(os.path.join(golden_dir, "generator.npz"))
    g = _fresh_generator(env)
    mel, face = O.make_generator_inputs(3, seed=2)
    with torch.no_grad():
        y = g(mel.cuda(), face.cuda()).cpu().numpy()
    assert np.abs(y - gold["gen4n3_out"]).max() <= 8e-3      # stress weights, see test_gpu_nets.py
    assert np.abs(y - gold["gen4n3_out"]).mean() <= 6e-4


def test_variants_agree_with_each_other():
    """Different tilings / kernels, same arithmetic up to fp32 summation order and one fp16 rounding per block."""
    mel, face = O.make_generator_inputs(4, seed=6)
    outs = []
    for env in ({}, {k: "1" for k in FLAGS}):
        g = _fresh_generator(env)
        with torch.no_grad():
            outs.append(g(mel.cuda(), face.cuda()).cpu())
    # each is within ~4e-3 of the fp32 reference on these stress weights (fp16 rounding points differ per tiling)
    assert (outs[0] - outs[1]).abs().max().item() <= 8e-3
    assert (outs[0] - outs[1]).abs().mean().item() <= 4e-4


@pytest.mark.parametrize("B,T", [(5, 0), (70, 0), (3, 5), (67, 2)])
def test_host_entry_point_matches_device_path(B, T):
    from wav2lip_b200 import _lib
    g = _fresh_generator({})
    mel, face = O.make_generator_inputs(B, seed=B, t=T if T > 0 else None)
    with torch.no_grad():
        y_dev = g(mel.cuda(), face.cuda()).cpu()
    ctx = g._w2l_ctx
    mel_h, face_h = mel.contiguous().pin_memory(), face.contiguous().pin_memory()
    out_h = torch.empty_like(y_dev).pin_memory()
    _lib.check(ctx.lib.w2l_generator_forward_host(ctx.h, C.c_void_p(mel_h.data_ptr()), C.c_void_p(face_h.data_ptr()),
                                                  C.c_void_p(out_h.data_ptr()), B, T))
    assert torch.equal(out_h, y_dev)
    # pageable (non-pinned) host memory works too
    out_p = torch.empty_like(y_dev)
    _lib.check(ctx.lib.w2l_generator_forward_host(ctx.h, C.c_void_p(mel.contiguous().data_ptr()),
                                                  C.c_void_p(face.contiguous().data_ptr()), C.c_void_p(out_p.data_ptr()), B, T))
    assert torch.equal(out_p, y_dev)


def test_submit_wait_pipeline_matches_device_path():
    """w2l_generator_submit_host / _submit_u8_host + w2l_host_wait: results land in submission order and equal the
    device path bit for bit, across changing batch sizes (staging buffers grow -> the pipeline drains first)."""
    from wav2lip_b200 import _lib
    import ctypes as C
    g = _fresh_generator({})
    ctx = g._w2l_ctx
    sizes = [3, 70, 5, 5, 130, 1]
    batches, refs, outs = [], [], []
    for i, n in enumerate(sizes):
        mel, face = O.make_generator_inputs(n, seed=100 + i)
        with torch.no_grad():
            refs.append(g(mel.cuda(), face.cuda()).cpu())
        batches.append((mel.contiguous().pin_memory(), face.contiguous().pin_memory()))
        outs.append(torch.zeros_like(refs[-1]).pin_memory())
    done = 0
    for i, n in enumerate(sizes):
        _lib.check(ctx.lib.w2l_generator_submit_host(ctx.h, C.c_void_p(batches[i][0].data_ptr()), C.c_void_p(batches[i][1].data_ptr()),
                                                     C.c_void_p(outs[i].data_ptr()), n, 0))
        _lib.check(ctx.lib.w2l_host_wait(ctx.h, 1))
        while done < i:   # everything but the newest submission is complete
            assert torch.equal(outs[done], refs[done]), done
            done += 1
    _lib.check(ctx.lib.w2l_host_wait(ctx.h, 0))
    assert torch.equal(outs[-1], refs[-1])
    # three submissions without a wait: the third one retires the first by itself
    for o in outs[:3]:
        o.zero_()
    for i in range(3):
        _lib.check(ctx.lib.w2l_generator_submit_host(ctx.h, C.c_void_p(batches[i][0].data_ptr()), C.c_void_p(batches[i][1].data_ptr()),
                                                     C.c_void_p(outs[i].data_ptr()), sizes[i], 0))
    _lib.check(ctx.lib.w2l_host_wait(ctx.h, 0))
    for i in range(3):
        assert torch.equal(outs[i], refs[i])
    # a synchronous call after asynchronous ones
    _lib.check(ctx.lib.w2l_generator_submit_host(ctx.h, C.c_void_p(batches[1][0].data_ptr()), C.c_void_p(batches[1][1].data_ptr()),
                                                 C.c_void_p(outs[1].data_ptr()), sizes[1], 0))
    o2 = torch.zeros_like(refs[4]).pin_memory()
    _lib.check(ctx.lib.w2l_generator_forward_host(ctx.h, C.c_void_p(batches[4][0].data_ptr()), C.c_void_p(batches[4][1].data_ptr()),
                                                  C.c_void_p(o2.data_ptr()), sizes[4], 0))
    assert torch.equal(o2, refs[4]) and torch.equal(outs[1], refs[1])


def test_infer_stream_fp32_and_u8():
    g = _fresh_generator({})
    gen = torch.Generator().manual_seed(5)
    f32 = [O.make_generator_inputs(n, seed=200 + n) for n in (4, 9, 2)]
    with torch.no_grad():
        refs = [g(m.cuda(), f.cuda()).cpu() for m, f in f32]
    got = list(g.infer_stream(iter(f32)))
    assert len(got) == 3 and all(torch.equal(a, b) for a, b in zip(got, refs))
    u8 = [((torch.rand((n, 1, 80, 16), generator=gen) * 8 - 4), torch.randint(0, 256, (n, 96, 96, 3), generator=gen, dtype=torch.uint8))
          for n in (6, 1, 11)]
    with torch.no_grad():
        refs8 = [g.infer_u8(m.cuda(), f.cuda()).cpu() for m, f in u8]
    got8 = list(g.infer_stream(iter(u8)))
    assert len(got8) == 3 and all(torch.equal(a, b) for a, b in zip(got8, refs8))
    assert list(g.infer_stream(iter([]))) == []


def test_launch_counter_and_profile():
    from wav2lip_b200 import _lib
    g = _fresh_generator({})
    mel, face = O.make_generator_inputs(2, 0)
    ctx = g._w2l_ctx
    with torch.no_grad():
        g(mel.cuda(), face.cuda())
        n0 = ctx.launch_count()
        g(mel.cuda(), face.cuda())
        n1 = ctx.launch_count()
    per_forward = n1 - n0
    assert 50 <= per_forward <= 80          # 2 ingest + one launch per block (4 per generic transposed conv)
    prof = ctx.profile_plan(_lib.NET_GENERATOR, iters=1)
    assert len(prof) == per_forward - 2
    total_flop = sum(f for _, _, f in prof)
    assert abs(total_flop / (2 * 2 * 3966984192) - 1) < 0.001  # = 2 crops x 7.934 GFLOP minus the fused 1x1 head
    assert ctx.device_bytes() > 70e6   # >= the packed 16-bit weights (36.3 M params)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_two_devices_in_one_process():
    """One context per device in the same process (kernel attributes are per device): same inputs, same bits."""
    from wav2lip_b200.models import Wav2Lip
    sd = O.make_state_dict("generator", 0)
    mel, face = O.make_generator_inputs(5, seed=3)
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        g = Wav2Lip()
        g.load_state_dict(sd, strict=True)
        g = g.to(dev).eval()
        with torch.no_grad():
            outs.append(g(mel.to(dev), face.to(dev)).cpu())
    assert torch.equal(outs[0], outs[1])
