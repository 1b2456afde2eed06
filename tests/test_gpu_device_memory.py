"""Device memory of a context: a failed allocation leaves the context usable, and w2l_device_bytes counts every block the
context holds — weights once however often they are reloaded, the private plans of the single-block entries only while
those run, and the training plans while they exist."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import w2l_oracle as O

pytestmark = pytest.mark.gpu

P = lambda t: C.c_void_p(t.data_ptr())


def _generator():
    from wav2lip_b200.models import Wav2Lip
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0), strict=True)
    return g.cuda().eval()


def test_failed_allocation_leaves_the_context_usable():
    """An oversized w2l_lipsync_frames_u8 (its crop buffer alone is larger than the card) fails with W2L_ENOMEM without
    reserving anything; the next, normal call on the same context succeeds and matches a fresh context bit for bit."""
    from wav2lip_b200 import _lib
    g = _generator()
    frames = torch.randint(0, 256, (1, 96, 96, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(0)).cuda()
    ctx = g._ensure(frames)
    n_big = torch.cuda.get_device_properties(0).total_memory // (96 * 96 * 3) + 1
    boxes = np.tile(np.array([[0, 0, 96, 0, 96]], dtype=np.int32), (n_big, 1))
    mel = torch.zeros((2, 1, 80, 16), device="cuda")
    out = torch.empty((2, 96, 96, 3), device="cuda", dtype=torch.uint8)
    torch.cuda.synchronize()
    rc = ctx.lib.w2l_lipsync_frames_u8(ctx.h, P(mel), P(frames), 1, 96, 96, boxes.ctypes.data_as(C.POINTER(C.c_int32)), n_big,
                                       P(out), None)
    assert rc == _lib.W2L_ENOMEM, (rc, ctx.lib.w2l_last_error())

    mel2, _ = O.make_generator_inputs(2, 0)
    boxes2 = [[0, 0, 96, 0, 96], [0, 10, 80, 5, 90]]
    with torch.no_grad():
        got = g.infer_frames(mel2.cuda(), frames, boxes2)
        ref = _generator().infer_frames(mel2.cuda(), frames, boxes2)
    assert torch.equal(got, ref)


def test_reloading_weights_keeps_device_bytes():
    from wav2lip_b200 import _lib
    ctx = _lib.Context(0, _lib.PREC_F16)
    sd = {k: v.cuda().contiguous() for k, v in O.make_state_dict("generator", 0).items() if v.dtype.is_floating_point}
    tensors = {k: (v.data_ptr(), v.numel()) for k, v in sd.items()}
    ctx.load_weights(_lib.NET_GENERATOR, tensors)
    loaded = ctx.device_bytes()
    ctx.load_weights(_lib.NET_GENERATOR, tensors)
    assert ctx.device_bytes() == loaded


def test_single_block_entries_release_what_they_allocate():
    """w2l_conv_block_forward and w2l_conv_block_train build a private plan and weights per call and free them on return.
    (The first training call also allocates the context's persistent training scratch, so each entry runs once first.)"""
    from wav2lip_b200 import _lib
    ctx = _lib.Context(0, _lib.PREC_BF16)
    g = torch.Generator().manual_seed(1)
    n, c, h, w = 2, 64, 12, 12
    li = _lib.LayerInfo()
    li.name = b"block"
    li.kind = _lib.BLOCK_CONV_BN_RELU
    li.cin, li.cout, li.kh, li.kw, li.sh, li.sw, li.ph, li.pw = c, c, 3, 3, 1, 1, 1, 1
    li.out_pad, li.residual = 0, 1
    t = lambda *s: torch.randn(s, generator=g).cuda()
    x, wt, b, dy = t(n, c, h, w), t(c, c, 3, 3) / 24, t(c), t(n, c, h, w)
    gamma, beta, mean, var = 1 + 0.1 * t(c), t(c), t(c), 1 + torch.rand(c, generator=g).cuda()
    y, dx, dw = torch.empty_like(x), torch.empty_like(x), torch.empty_like(wt)
    db, dgamma, dbeta = torch.empty_like(b), torch.empty_like(b), torch.empty_like(b)

    def forward():
        _lib.check(ctx.lib.w2l_conv_block_forward(ctx.h, C.byref(li), P(x), n, h, w, P(wt), P(b), P(gamma), P(beta), P(mean),
                                                  P(var), P(y), None))

    def train():
        _lib.check(ctx.lib.w2l_conv_block_train(ctx.h, C.byref(li), P(x), n, h, w, P(wt), P(b), P(gamma), P(beta), P(mean),
                                                P(var), P(dy), P(y), P(dx), P(dw), P(db), P(dgamma), P(dbeta), None))

    for entry in (forward, train):
        entry()
        before = ctx.device_bytes()
        entry()
        assert ctx.device_bytes() == before, entry.__name__


def test_training_plans_are_counted():
    """A generator training step at B = 16, T = 5 holds at least the decoder's skip-concat buffers and their gradients
    (wav2lip.py:108; widths of GeneratorSpec in netspec.h), and rebinding the generator drops them again."""
    from wav2lip_b200.models import Wav2Lip
    from wav2lip_b200.training import Wav2LipTrainStep
    B, T = 16, 5
    hw = [1, 3, 6, 12, 24, 48, 96]
    dec_c = [512, 512, 512, 384, 256, 128, 64]
    skip_c = [512, 512, 256, 128, 64, 32, 16]
    concat = B * T * sum(s * s * (d + k) for s, d, k in zip(hw, dec_c, skip_c)) * 2 * 2   # bf16, value + gradient
    model = Wav2Lip()
    model.load_state_dict(O.make_state_dict("generator", 0, init="default"), strict=True)
    model = model.cuda().train()
    step = Wav2LipTrainStep(model, None, syncnet_wt=0.0)
    ctx = step.b.ctx
    g = torch.Generator().manual_seed(0)
    indiv_mels, x = O.make_generator_inputs(B, seed=0, t=T)
    gt = torch.rand((B, 3, T, 96, 96), generator=g)
    before = ctx.device_bytes()
    step(x.cuda(), indiv_mels.cuda(), None, gt.cuda())
    torch.cuda.synchronize()
    with_plan = ctx.device_bytes()
    assert with_plan - before >= concat, (with_plan - before, concat)
    step.b.key = None   # the binding's tensors are bound again: w2l_train_bind drops the net's plans and Adam moments
    step.b.ensure()
    assert with_plan - ctx.device_bytes() >= concat, (with_plan - ctx.device_bytes(), concat)
