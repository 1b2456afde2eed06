"""Training parity: every backward launch of the three networks' training plans, block by block, against float64
recomputed from the GPU's own tape.

After one train-mode forward + backward (default-init weights, random inputs and output gradients), each block's tape
is read back through w2l_debug_train_tensor (x, z, y, dy, dz, du, dx, dx_add and the batch statistics, exactly the
stored bf16 / fp32 values) and every quantity the block computed is recomputed in float64 on the GPU (float64 never
takes the TF32 path) from the tape and bf16(W).  Feeding each step the GPU's own inputs takes the ~1e5 amplification
of batch-statistics BatchNorm (DESIGN section 7) out of the comparison, so every block of the real networks at real
shapes is held to a bar derived from its arithmetic.  ulp16 / ACC = 2^-16 / the mean-rounding check are the ones of
tests/test_gpu_kernel_parity.py; M = pixels of the block output; sums run over the batch and the pixels.

  quantity          float64 reference                                     bar per element
  z (bf16)          conv(x, bf16 W)                                       ulp16 + ACC * conv(|x|, |W|)
  mean, invstd      sum z / M, (sum z^2 / M - mean^2 + eps)^-1/2          ACC * sum|z| / M;  invstd * (ACC/2 * (sum z^2 + 2|mean| sum|z|)
                                                                          / M / (var + eps) + 2^-23)
  y (bf16)          relu(G z + beta - mean G [+ x]), G = fp32(gamma invstd)   ulp16 + ACC * (|G z| + |beta| + |mean G| + |x|)
                    with the GPU's mean / invstd; nonorm: lrelu(conv + b)      (nonorm: ACC * (conv(|x|,|W|) + |b|))
  dz (bf16)         c1 (du - S/M - zhat * invstd (Q - mean S) / M),      ulp16 + ACC * |c1| (|du| + A/M + invstd^2 (|z| + |mean|)
                    du = dy * (y > 0), S = sum du, Q = sum du z              * (B + |mean| A) / M),  A = sum|du|, B = sum|du z|
                    nonorm: dy * (y > 0 ? 1 : 0.01)                       ulp16 + ACC * |dz|
  du (bf16)         dy * (y > 0)                                          exact
  dbeta, dgamma     S, invstd (Q - mean S);  nonorm db = sum dz           ACC * A, ACC * invstd (B + |mean| A);  ACC * sum|dz|
  conv bias grad    0 under a BatchNorm                                   exact
  dx (bf16)         dgrad(dz, bf16 W) + du / + dx_add                     ulp16 + ACC * (dgrad(|dz|, |W|) + |add|)
  dW (fp32)         wgrad(x, dz)                                          max(ACC, L * 2^-24) * wgrad(|x|, |dz|)
  running mean/var  0.9 old + 0.1 (mean + b), 0.9 old + 0.1 var m/(m-1)   2^-20 * (0.9 |old| + 0.1 |new term|)
                    with var = invstd^-2 - eps from the GPU's stats

The bf16 bars are the inference file's: one rounding flip plus 2^-16 of the magnitude sum for fp32 accumulation.  The
dz bar takes its magnitude from the absolute values of every term the kernels sum (the coefficients come from fp32
partial sums of du and du*z, whose difference Q - mean S cancels), not from |P du| + |Q z| + |R|, which the cancellation
can make arbitrarily small.  The dW bar is derived, not fitted: a wgrad unit accumulates its share of the pixels in
fp32 registers, P/16 wgmma k-steps per K chunk over ceil(chunks/splits) chunks, and the reduction adds `splits` more
partial sums, so one output element's fp32 add chain is L = ceil(chunks/splits) * P/16 + splits long, and its rounding
error is at most L * 2^-24 of the magnitude sum.  The forward's bar 2^-16 = 256 * 2^-24 already covers chains of up to
256 adds; beyond that the bar grows with L.  A dropped split costs about 1/splits of the magnitude and a dropped
128-pixel chunk 128/M of it, both far above either term.  Every bf16 store with >= 1e4 elements also passes the mean
signed rounding check (|bias| <= 0.05 ulp; a truncating conversion gives about -0.5).

Besides the tape parity: forward + backward twice gives bit-identical gradients, input gradient and running
statistics (the split-K reduction has no atomics); the switches that only move launches between streams or keep the
K order (W2L_DISABLE_WGSTREAM / AUXSTREAM / PDL / MT2 / TMAEPI / SIDESTREAM) give bit-identical training outputs;
the switches that change kernels (HALO / FOLD / CTFUSED) are checked with the tape parity on the blocks whose kernels
change; W2L_TRAIN_ACCUMULATE adds exactly fp32(G1 + G2) to every bound gradient; W2L_TRAIN_NO_STAT_UPDATE leaves the
running statistics bit-unchanged; and a coverage test fails if some wgrad instantiation, wgrad form, tap-group / tile /
split-K shape or dgrad form is reached by no checked block.

Measured on one H100 SXM (80 GB, 700 W); the file takes about 45 s there.  Over all blocks of the four network runs:
mean 0.00, invstd 0.01, dgamma / dbeta 0.00, nonorm db 0.01, running mean 0.15, running var 0.10 of their bars; du and the
conv bias under a BatchNorm exact.  Under W2L_DISABLE_HALO (15 blocks change kernel), _FOLD (2) and _CTFUSED (1) the
changed blocks stay within the same maxima.  Per block, max err/bar (blank: exactly 0, or the block has no such tensor):
  network / block                          z     y    dz    dx    dW
  gen audio_encoder.0                                0.00        0.01
  gen audio_encoder.1                    0.99  0.57  0.99  0.98  0.02
  gen audio_encoder.2                    0.98  0.01  0.00  0.98  0.02
  gen audio_encoder.3                    0.95        0.18  0.99  0.03
  gen audio_encoder.4                    0.98              0.99  0.03
  gen audio_encoder.5                    0.97  0.99  0.99  0.99  0.02
  gen audio_encoder.6                    0.96  0.01  0.02  0.99  0.02
  gen audio_encoder.7                    0.98  0.04        0.97  0.02
  gen audio_encoder.8                    0.97        0.36  0.96  0.02
  gen audio_encoder.9                    0.97              0.04  0.01
  gen audio_encoder.10                   0.55        0.99  0.02  0.01
  gen audio_encoder.11                   0.94              0.89  0.01
  gen audio_encoder.12                                           0.01
  gen face_encoder_blocks.0.0            0.98        0.99        0.02
  gen face_encoder_blocks.1.0            0.99        0.19  0.99  0.02
  gen face_encoder_blocks.1.1            0.98  0.43  0.00  0.99  0.02
  gen face_encoder_blocks.1.2            0.99  0.98  1.00  0.99  0.01
  gen face_encoder_blocks.2.0            0.99        0.06  0.99  0.05
  gen face_encoder_blocks.2.1            0.98  0.78  0.01  0.98  0.04
  gen face_encoder_blocks.2.2            0.99  0.99  0.99  0.99  0.03
  gen face_encoder_blocks.2.3            0.99  0.84  0.95  0.97  0.03
  gen face_encoder_blocks.3.0            0.98  0.97  1.00  0.96  0.05
  gen face_encoder_blocks.3.1            0.95  0.99        0.96  0.04
  gen face_encoder_blocks.3.2            0.95  0.08        0.98  0.03
  gen face_encoder_blocks.4.0            0.96  0.01  0.98  0.94  0.02
  gen face_encoder_blocks.4.1            0.97              0.95  0.02
  gen face_encoder_blocks.4.2            0.97  0.02  0.00  0.97  0.02
  gen face_encoder_blocks.5.0            0.97              0.97  0.02
  gen face_encoder_blocks.5.1            0.95  0.96  0.86  0.96  0.01
  gen face_encoder_blocks.6.0            0.91        0.00  0.99  0.01
  gen face_encoder_blocks.6.1                                    0.01
  gen face_decoder_blocks.0.0                              0.23  0.01
  gen face_decoder_blocks.1.0            0.02              0.90  0.01
  gen face_decoder_blocks.1.1            0.87              0.97  0.02
  gen face_decoder_blocks.2.0            0.96  0.21  0.03  0.96  0.02
  gen face_decoder_blocks.2.1            0.97        0.99  0.97  0.02
  gen face_decoder_blocks.2.2            0.97  0.02        0.97  0.02
  gen face_decoder_blocks.3.0            0.98        0.99  0.97  0.07
  gen face_decoder_blocks.3.1            0.98  0.51  0.00  0.97  0.05
  gen face_decoder_blocks.3.2            0.98  0.65  0.97  0.98  0.03
  gen face_decoder_blocks.4.0            0.98  0.02  0.49  0.98  0.13
  gen face_decoder_blocks.4.1            0.99  1.00  0.99  0.98  0.06
  gen face_decoder_blocks.4.2            0.98  0.99  0.31  0.98  0.04
  gen face_decoder_blocks.5.0            0.99  0.00  1.00  0.98  0.31
  gen face_decoder_blocks.5.1            0.98  0.99  1.00  0.99  0.02
  gen face_decoder_blocks.5.2            0.99  0.95  1.00  0.99  0.02
  gen face_decoder_blocks.6.0            0.99  0.99  1.00  0.99  0.11
  gen face_decoder_blocks.6.1            0.99  1.00  0.99  0.99  0.01
  gen face_decoder_blocks.6.2            0.99  1.00  1.00  0.99  0.01
  gen output_block.0                     0.99        0.99  0.99  0.02
  sync audio_encoder.0                               0.03        0.01
  sync audio_encoder.1                   0.98  0.97  0.98  0.99  0.02
  sync audio_encoder.2                   0.99  0.03  0.49  0.99  0.02
  sync audio_encoder.3                   0.96        0.99  0.99  0.03
  sync audio_encoder.4                   0.98  0.38        0.99  0.03
  sync audio_encoder.5                   0.97  0.04  0.99  0.98  0.02
  sync audio_encoder.6                   0.96  0.00  0.99  0.99  0.03
  sync audio_encoder.7                   0.97  0.12  0.00  0.97  0.03
  sync audio_encoder.8                   0.97        0.00  0.98  0.03
  sync audio_encoder.9                   0.96              0.97  0.02
  sync audio_encoder.10                  0.96  1.00  0.00  0.98  0.02
  sync audio_encoder.11                  0.94              0.96  0.01
  sync audio_encoder.12                  0.96  0.98        0.98  0.01
  sync audio_encoder.13                  0.05              0.04  0.01
  sync face_encoder.0                    0.98  1.00  0.99  0.98  0.01
  sync face_encoder.1                    0.98  1.00  0.99  0.99  0.02
  sync face_encoder.2                    0.99  1.00  1.00  0.99  0.01
  sync face_encoder.3                    0.99  1.00  0.99  0.99  0.01
  sync face_encoder.4                    0.98        0.99  0.99  0.02
  sync face_encoder.5                    0.99  0.99  1.00  0.99  0.02
  sync face_encoder.6                    0.99  0.94  0.89  0.99  0.02
  sync face_encoder.7                    0.99  0.82  0.69  0.99  0.02
  sync face_encoder.8                    0.99  0.84  0.00  0.99  0.05
  sync face_encoder.9                    0.98  0.88  0.99  0.98  0.05
  sync face_encoder.10                   0.97  1.00  0.99  0.98  0.06
  sync face_encoder.11                   0.98  0.43  0.00  0.99  0.03
  sync face_encoder.12                   0.96  0.09  0.95  0.97  0.03
  sync face_encoder.13                   0.97  0.56        0.98  0.03
  sync face_encoder.14                   0.97        0.00  0.99  0.03
  sync face_encoder.15                   0.95              0.97  0.01
  sync face_encoder.16                   0.46              0.22  0.01
  disc face_encoder_blocks.0.0                 0.99        0.98  0.02
  disc face_encoder_blocks.1.0                 0.99        0.99  0.06
  disc face_encoder_blocks.1.1                 0.98        0.98  0.06
  disc face_encoder_blocks.2.0                 0.99        0.99  0.17
  disc face_encoder_blocks.2.1                 0.98        0.98  0.12
  disc face_encoder_blocks.3.0                 0.99        0.99  0.12
  disc face_encoder_blocks.3.1                 0.98        0.98  0.16
  disc face_encoder_blocks.4.0                 0.98        0.99  0.07
  disc face_encoder_blocks.4.1                 0.98        0.97  0.07
  disc face_encoder_blocks.5.0                 0.98        0.99  0.02
  disc face_encoder_blocks.5.1                 0.97        0.96  0.04
  disc face_encoder_blocks.6.0                 0.76        0.97  0.01
  disc face_encoder_blocks.6.1                             0.94
  disc, no input grad face_encoder_blocks.0.0       0.99              0.02
"""
import ctypes as C
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import w2l_oracle as O
from test_gpu_kernel_parity import ACC, BF16, ulp16

pytestmark = pytest.mark.gpu

SWITCHES = ["W2L_DISABLE_WGSTREAM", "W2L_DISABLE_AUXSTREAM", "W2L_DISABLE_PDL", "W2L_DISABLE_MT2", "W2L_DISABLE_TMAEPI",
            "W2L_DISABLE_SIDESTREAM", "W2L_DISABLE_HALO", "W2L_DISABLE_FOLD", "W2L_DISABLE_CTFUSED", "W2L_DISABLE_FOLDS2"]
BIT_IDENTICAL = SWITCHES[:6]
KERNEL_CHOICE = ["W2L_DISABLE_HALO", "W2L_DISABLE_FOLD", "W2L_DISABLE_CTFUSED"]
WGRAD, ACCUMULATE, INPUT_GRAD, NO_STAT_UPDATE = 1, 2, 4, 8
GEN, SYNC, DISC = 0, 1, 2
NET_NAME = {GEN: "generator", SYNC: "syncnet", DISC: "disc"}
U24 = 2.0 ** -24
RUN_BAR = 2.0 ** -20

# ------------------------------------------------------------------------------------------------------------------
# contexts: one per switch set, created with the switches in the environment, closed at module teardown
# ------------------------------------------------------------------------------------------------------------------
_CTX = {}


def _ctx(off=()):
    from wav2lip_b200 import _lib
    key = tuple(sorted(off))
    if key not in _CTX:
        old = {k: os.environ.get(k) for k in SWITCHES}
        try:
            for k in SWITCHES:
                os.environ.pop(k, None)
            for k in off:
                os.environ[k] = "1"
            _CTX[key] = _lib.Context(0, _lib.PREC_BF16)   # the W2L_DISABLE_* switches are read here
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    return _CTX[key]


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in _CTX.values():
        c.close()
    _CTX.clear()


# ------------------------------------------------------------------------------------------------------------------
# one training forward + backward of a network through the C ABI
# ------------------------------------------------------------------------------------------------------------------
P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class NetRun:
    """Bound fp32 parameters / gradients of one network on one context, and its fixed inputs."""

    def __init__(self, ctx, net, B, T, seed=0):
        self.ctx, self.net, self.B, self.T = ctx, net, B, T
        sd = O.make_state_dict(NET_NAME[net], seed, init="default")
        self.sd = {k: v for k, v in sd.items() if v.dtype.is_floating_point}
        self.val = {k: v.to("cuda", torch.float32).contiguous() for k, v in self.sd.items()}
        self.grad = {k: torch.zeros_like(v) for k, v in self.val.items() if "running" not in k}
        names = list(self.val)
        n = len(names)
        arr_n = (C.c_char_p * n)(*[k.encode() for k in names])
        arr_v = (C.c_void_p * n)(*[self.val[k].data_ptr() for k in names])
        arr_g = (C.c_void_p * n)(*[self.grad[k].data_ptr() if k in self.grad else None for k in names])
        arr_c = (C.c_int64 * n)(*[self.val[k].numel() for k in names])
        torch.cuda.synchronize()
        from wav2lip_b200 import _lib
        _lib.check(ctx.lib.w2l_train_bind(ctx.h, net, n, arr_n, arr_v, arr_g, arr_c))
        g = torch.Generator().manual_seed(100 + seed)
        if net == GEN:
            mel, face = O.make_generator_inputs(B, seed=seed)
            self.ins = [mel.cuda().contiguous(), face.cuda().contiguous()]
            self.outs = [torch.empty((B, 3, 96, 96), device="cuda"), None]
            self.dout = [torch.randn((B, 3, 96, 96), generator=g).cuda(), None]
            self.dinput = None
        elif net == SYNC:
            mel, face = O.make_syncnet_inputs(B, seed=seed)
            self.ins = [mel.cuda().contiguous(), face.cuda().contiguous()]
            self.outs = [torch.empty((B, 512), device="cuda"), torch.empty((B, 512), device="cuda")]
            self.dout = [torch.randn((B, 512), generator=g).cuda(), torch.randn((B, 512), generator=g).cuda()]
            self.dinput = torch.empty((B, 15, 48, 96), device="cuda")
        else:
            self.ins = [O.make_disc_inputs(B, T, seed=seed).cuda().contiguous(), None]
            self.outs = [torch.empty((B * T, 1), device="cuda"), None]
            self.dout = [torch.randn((B * T, 1), generator=g).cuda(), None]
            self.dinput = torch.empty((B, 3, T, 96, 96), device="cuda")

    def running(self):
        return {k: v.clone() for k, v in self.val.items() if "running" in k}

    def forward(self, flags):
        from wav2lip_b200 import _lib
        _lib.check(self.ctx.lib.w2l_train_forward(self.ctx.h, self.net, P(self.ins[0]), P(self.ins[1]), P(self.outs[0]),
                                                  P(self.outs[1]), self.B, self.T, flags, None))

    def backward(self, flags, dout=None):
        from wav2lip_b200 import _lib
        d = dout or self.dout
        di = self.dinput if flags & INPUT_GRAD else None
        _lib.check(self.ctx.lib.w2l_train_backward(self.ctx.h, self.net, P(d[0]), P(d[1]), P(di), flags & ~INPUT_GRAD,
                                                   None))
        torch.cuda.synchronize()

    def step(self, flags):
        """forward + backward; returns every training output (gradients, input gradient, running statistics, outputs)"""
        self.forward(flags)
        self.backward(flags)
        out = {"grad." + k: v.clone() for k, v in self.grad.items()}
        out.update({"run." + k: v for k, v in self.running().items()})
        out.update({f"out{i}": o.clone() for i, o in enumerate(self.outs) if o is not None})
        if flags & INPUT_GRAD:
            out["dinput"] = self.dinput.clone()
        return out


NET_CASES = {   # (net, B, T, flags)
    "generator": (GEN, 4, 0, WGRAD),
    "syncnet": (SYNC, 8, 0, WGRAD | INPUT_GRAD),
    "disc-input-grad": (DISC, 2, 5, WGRAD | INPUT_GRAD),
    "disc": (DISC, 2, 5, WGRAD),
}


# ------------------------------------------------------------------------------------------------------------------
# float64 references of one block, from its tape
# ------------------------------------------------------------------------------------------------------------------
def bf16(t):
    return t.to(torch.bfloat16).double()


def _geom(b):
    return (b["kh"], b["kw"]), (b["sh"], b["sw"]), (b["ph"], b["pw"])


def conv_fwd(b, x, w):
    k, s, p = _geom(b)
    if b["kind"] == 1:
        return F.conv_transpose2d(x, w, stride=s, padding=p, output_padding=b["out_pad"])
    return F.conv2d(x, w, stride=s, padding=p)


def conv_dgrad(b, dz, w):
    k, s, p = _geom(b)
    if b["kind"] == 1:
        return F.conv2d(dz, w, stride=s, padding=p)
    return torch.nn.grad.conv2d_input((dz.shape[0], b["cin"], b["h_in"], b["w_in"]), w, dz, stride=s, padding=p)


def conv_wgrad(b, x, dz):
    k, s, p = _geom(b)
    if b["kind"] == 1:   # dW[ci][co][r][s] = sum x[ci] * dz[co] at the strided, tap-shifted position: the conv of dz
        return torch.nn.grad.conv2d_weight(dz, (b["cin"], b["cout"]) + k, x, stride=s, padding=p)
    return torch.nn.grad.conv2d_weight(x, (b["cout"], b["cin"]) + k, dz, stride=s, padding=p)


class Checker:
    """err/bar bookkeeping: check() raises on the first element above its bar."""

    def __init__(self, what):
        self.what, self.worst = what, {}

    def check(self, q, got, ref, bar, bf16_store=False, sel_mag=None):
        got = got.to(ref.device, torch.float64)
        assert got.shape == ref.shape, (self.what, q, tuple(got.shape), tuple(ref.shape))
        assert torch.isfinite(got).all(), f"{self.what} {q}: non-finite values"
        err = (got - ref).abs()
        if bf16_store:
            bar = bar + ulp16(torch.maximum(got.abs(), ref.abs()), BF16)
        ratio = (err / bar).max().item() if ref.numel() else 0.0
        if ratio > 1.0:
            i = int(torch.argmax(err / bar))
            idx = tuple(int(t) for t in torch.unravel_index(torch.tensor(i), ref.shape))
            raise AssertionError(f"{self.what} {q}: max err/bar {ratio:.3g} at {idx}: got {got.flatten()[i].item():.9g} "
                                 f"ref {ref.flatten()[i].item():.9g} bar {bar.flatten()[i].item():.3g}")
        if bf16_store and ref.numel() >= 10_000:
            sel = ref.abs() > sel_mag if sel_mag is not None else ref != 0
            bias = (torch.sign(ref[sel]) * (got[sel] - ref[sel]) / ulp16(ref[sel], BF16)).mean().item()
            assert abs(bias) <= 0.05, f"{self.what} {q}: rounding bias {bias:.4f} ulp (round-to-nearest gives ~0)"
        self.worst[q] = max(self.worst.get(q, 0.0), ratio)
        return ratio

    def exact(self, q, got, ref):
        assert torch.equal(got.to(ref.device, ref.dtype), ref), f"{self.what} {q}: not exact"
        self.worst.setdefault(q, 0.0)


def wgrad_chain(b):
    """fp32 add chain of one dW element: ceil(chunks / splits) * P/16 wgmma k-steps + the split-K sum"""
    return math.ceil(b["wg_chunks"] / b["wg_splits"]) * b["wg_p"] // 16 + b["wg_splits"]


def check_block(run, k, b, chk, old_run):
    """Every quantity of block k (forward order) of the last training step of `run`, from its tape."""
    from wav2lip_b200 import _lib
    ctx, net = run.ctx, run.net
    tape = lambda which: ctx.train_tensor(net, k, which)
    name = b["name"]
    chk.what = f"{NET_NAME[net]} {name}"
    W = bf16(run.val[f"{name}.conv_block.0.weight"].double())
    bias = run.val[f"{name}.conv_block.0.bias"].double()
    x = tape(_lib.TAPE_X).double()
    y = tape(_lib.TAPE_Y).double()
    dy = tape(_lib.TAPE_DY).double()
    dz = tape(_lib.TAPE_DZ).double()
    c4 = lambda t: t.view(1, -1, 1, 1)
    s_all = (0, 2, 3)
    mag_conv = conv_fwd(b, x.abs(), W.abs())
    if b["kind"] == 2:   # nonorm: bias + LeakyReLU in the conv epilogue, dz = dy * slope, db = sum dz
        v = conv_fwd(b, x, W) + c4(bias)
        mag = mag_conv + c4(bias.abs())
        ref = bf16(F.leaky_relu(v, 0.01))
        chk.check("y", y, ref, ACC * mag, True, ACC * mag)
        dz_ref = dy * torch.where(y > 0, 1.0, 0.01)
        chk.check("dz", dz, bf16(dz_ref), ACC * dz_ref.abs(), True)
        if b["has_wgrad"]:
            chk.check("db", run.grad[f"{name}.conv_block.0.bias"].double(), dz_ref.sum(s_all),
                      ACC * dz_ref.abs().sum(s_all) + 1e-30)
        add = None
    else:
        z = tape(_lib.TAPE_Z).double()
        st = tape(_lib.TAPE_STATS).double()
        mean, istd = st[0].flatten(), st[1].flatten()
        zref = conv_fwd(b, x, W)
        chk.check("z", z, bf16(zref), ACC * mag_conv, True, ACC * mag_conv)
        M = z.numel() // z.shape[1]
        sz, sq, sa = z.sum(s_all), (z * z).sum(s_all), z.abs().sum(s_all)
        mean_ref = sz / M
        var_ref = (sq / M - mean_ref ** 2).clamp(min=0)
        chk.check("mean", mean, mean_ref, ACC * sa / M + 1e-30)
        istd_ref = (var_ref + 1e-5).rsqrt()
        chk.check("invstd", istd, istd_ref,
                  istd_ref * (ACC / 2 * (sq + 2 * mean_ref.abs() * sa) / M / (var_ref + 1e-5) + 2.0 ** -23))
        gamma, beta = run.val[f"{name}.conv_block.1.weight"], run.val[f"{name}.conv_block.1.bias"]
        G = (gamma * st[1].flatten().float()).double()          # fp32 product, as bn_finalize_kernel forms it
        Hs = beta.double() - mean * G
        v = c4(G) * z + c4(Hs)
        mag = (c4(G) * z).abs() + c4(beta.double().abs() + (mean * G).abs())
        if b["residual"]:
            v, mag = v + x, mag + x.abs()
        chk.check("y", y, bf16(F.relu(v)), ACC * mag, True, ACC * mag)
        # backward: du = dy * mask (the kernels' mask is y > 0, or G z + H > 0, which is the same test), sums, dz
        du = dy * (y > 0)
        if b["residual"]:
            chk.exact("du", tape(_lib.TAPE_DU).double(), du)
        S, Q = du.sum(s_all), (du * z).sum(s_all)
        A, Bm = du.abs().sum(s_all), (du * z).abs().sum(s_all)
        dg = istd * (Q - mean * S)
        c1 = gamma.double() * istd
        zhat = (z - c4(mean)) * c4(istd)
        dz_ref = c4(c1) * (du - c4(S / M) - zhat * c4(dg / M))
        dz_mag = c4(c1.abs()) * (du.abs() + c4(A / M) + c4(istd ** 2) * (z.abs() + c4(mean.abs())) * c4((Bm + mean.abs() * A) / M))
        chk.check("dz", dz, bf16(dz_ref), ACC * dz_mag, True, ACC * dz_mag)
        if b["has_wgrad"]:
            chk.check("dbeta", run.grad[f"{name}.conv_block.1.bias"].double(), S, ACC * A + 1e-30)
            chk.check("dgamma", run.grad[f"{name}.conv_block.1.weight"].double(), dg, ACC * istd * (Bm + mean.abs() * A) + 1e-30)
            chk.exact("dbias", run.grad[f"{name}.conv_block.0.bias"].double(), torch.zeros_like(S))
        rm, rv = f"{name}.conv_block.1.running_mean", f"{name}.conv_block.1.running_var"
        if old_run is not None and rm in old_run:
            o_m, o_v = old_run[rm].double(), old_run[rv].double()
            t_m = mean + bias
            var = istd ** -2 - 1e-5
            t_v = var * M / (M - 1)
            chk.check("running_mean", run.val[rm].double(), 0.9 * o_m + 0.1 * t_m, RUN_BAR * (0.9 * o_m.abs() + 0.1 * t_m.abs()) + 1e-30)
            chk.check("running_var", run.val[rv].double(), 0.9 * o_v + 0.1 * t_v,
                      RUN_BAR * (0.9 * o_v.abs() + 0.1 * (var.abs() + 1e-5) * M / (M - 1)))
        add = tape(_lib.TAPE_DU).double() if b["has_du"] else None
    if b["has_dx_add"]:
        add = tape(_lib.TAPE_DX_ADD).double()
    if b["has_dx"]:
        dx = tape(_lib.TAPE_DX).double()
        ref = conv_dgrad(b, dz, W)
        mag = conv_dgrad(b, dz.abs(), W.abs())
        if add is not None:
            ref, mag = ref + add, mag + add.abs()
        chk.check("dx", dx, bf16(ref), ACC * mag, True, ACC * mag)
    if b["has_wgrad"]:
        gw = run.grad[f"{name}.conv_block.0.weight"].double()
        ref = conv_wgrad(b, x, dz)
        mag = conv_wgrad(b, x.abs(), dz.abs())
        chk.check("dW", gw, ref, max(ACC, wgrad_chain(b) * U24) * mag + 1e-30)


_BLOCKS = {}   # case id -> block infos of the checked plans (coverage)
_RESULTS = {}  # (case id, switches) -> training outputs of one step


def tape_parity(case, off=(), only=None):
    net, B, T, flags = NET_CASES[case]
    ctx = _ctx(off)
    run = NetRun(ctx, net, B, T)
    old = run.running()
    _RESULTS[(case, tuple(sorted(off)))] = run.step(flags)
    blocks = ctx.train_blocks(net)
    assert blocks, case
    worst, per_block = {}, []
    for k, b in enumerate(blocks):
        if only is not None and b["name"] not in only:
            continue
        chk = Checker(case)
        check_block(run, k, b, chk, old)
        per_block.append(b["name"])
        print(f"BLOCK {case} {b['name']}: " + " ".join(f"{q} {v:.2f}" for q, v in chk.worst.items() if v > 0), flush=True)
        for q, v in chk.worst.items():
            worst[q] = max(worst.get(q, 0.0), v)
    return blocks, worst, per_block


def _report(what, worst):
    print(f"REPORT {what}: " + " ".join(f"{q} {v:.2f}" for q, v in sorted(worst.items())), flush=True)


@pytest.mark.parametrize("case", list(NET_CASES))
def test_tape_parity(case):
    blocks, worst, checked = tape_parity(case)
    _BLOCKS[case] = blocks
    _report(case, worst)
    assert len(checked) == len(blocks)


# ------------------------------------------------------------------------------------------------------------------
# single blocks through w2l_conv_block_train: shapes the networks do not reach
# ------------------------------------------------------------------------------------------------------------------
BLOCK_CASES = [   # (id, row, N, H, W)
    ("80 res: widened dgrad + du", O._c(80, 80, 3, 1, 1, True), 2, 24, 24),
    ("1x1 512 N=2048: two splits", O._c(512, 512, 1, 1, 0), 2048, 1, 1),
]


@pytest.mark.parametrize("case", BLOCK_CASES, ids=[c[0] for c in BLOCK_CASES])
def test_block_train_case(case):
    """w2l_conv_block_train on a shape the networks do not reach, against the float64 recipe with the kernels'
    rounding points of tests/test_gpu_train_blocks.py (its tape is not kept: that file's relative-L2 bar), and the
    block info it reports for the coverage test."""
    from wav2lip_b200 import _lib
    from test_gpu_train_blocks import REL, reference_same_rounding, rel_l2
    name, row, N, H, W = case
    kind, cin, cout, k, s, p, op, res = row
    (kh, kw), (sh, sw), (ph, pw) = O._pair(k), O._pair(s), O._pair(p)
    g = torch.Generator().manual_seed(N * 131 + cin)
    x = torch.randn((N, cin, H, W), generator=g)
    w = torch.randn((cout, cin, kh, kw), generator=g) / (cin * kh * kw) ** 0.5
    b0, gamma, beta = 0.1 * torch.randn(cout, generator=g), 1 + 0.2 * torch.randn(cout, generator=g), 0.1 * torch.randn(cout, generator=g)
    Ho, Wo = (H + 2 * ph - kh) // sh + 1, (W + 2 * pw - kw) // sw + 1
    dy = torch.randn((N, cout, Ho, Wo), generator=g)
    same = reference_same_rounding(x, w, b0, gamma, beta, dy, row)
    li = _lib.LayerInfo()
    li.name = b"block"
    li.kind = _lib.BLOCK_CONV_BN_RELU
    li.cin, li.cout, li.kh, li.kw, li.sh, li.sw, li.ph, li.pw, li.out_pad, li.residual = cin, cout, kh, kw, sh, sw, ph, pw, op, int(res)
    d = lambda t: t.float().contiguous().cuda()
    xd, wd, bd, gd, bed, dyd = map(d, (x, w, b0, gamma, beta, dy))
    yd, dxd, dwd = torch.empty((N, cout, Ho, Wo), device="cuda"), torch.empty_like(xd), torch.empty_like(wd)
    dbd, dgd, dbed = (torch.empty(cout, device="cuda") for _ in range(3))
    ctx = _ctx()
    _lib.check(ctx.lib.w2l_conv_block_train(ctx.h, C.byref(li), P(xd), N, H, W, P(wd), P(bd), P(gd), P(bed), None, None,
                                            P(dyd), P(yd), P(dxd), P(dwd), P(dbd), P(dgd), P(dbed), None))
    torch.cuda.synchronize()
    info = ctx.train_blocks(-1)
    assert len(info) == 1 and info[0]["name"] == "block" and info[0]["has_wgrad"] and info[0]["has_dx"], info
    _BLOCKS["block " + name] = info
    errs = {"y": rel_l2(yd.cpu(), same["y"]), "dx": rel_l2(dxd.cpu(), same["dx"]), "dw": rel_l2(dwd.cpu(), same["dw"]),
            "dgamma": rel_l2(dgd.cpu(), same["dgamma"]), "dbeta": rel_l2(dbed.cpu(), same["dbeta"])}
    print(f"REPORT block {name}: " + " ".join(f"{k} {v:.2e}" for k, v in errs.items())
          + f" splits {info[0]['wg_splits']} dgrad {[k['bn'] for k in info[0]['dgrad']]}", flush=True)
    assert all(v <= REL for v in errs.values()), errs
    assert dbd.abs().max().item() == 0.0


# ------------------------------------------------------------------------------------------------------------------
# determinism, switches, backward flags
# ------------------------------------------------------------------------------------------------------------------
def _diff(a, b):
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    return bad[:8], len(bad)


@pytest.mark.parametrize("case", list(NET_CASES))
def test_two_runs_bit_identical(case):
    net, B, T, flags = NET_CASES[case]
    run = NetRun(_ctx(), net, B, T)
    r1, r2 = run.step(flags | NO_STAT_UPDATE), run.step(flags | NO_STAT_UPDATE)
    bad = _diff(r1, r2)
    assert not bad[1], f"{case}: two runs differ in {bad}"


@pytest.mark.parametrize("flag", BIT_IDENTICAL)
@pytest.mark.parametrize("case", ["generator", "syncnet", "disc-input-grad"])
def test_switch_bit_identical(case, flag):
    """These switches move launches between streams or keep the K order of every sum: every training output
    (gradients, input gradient, running statistics, network outputs) is bit-identical to the default."""
    net, B, T, flags = NET_CASES[case]
    ref = NetRun(_ctx(), net, B, T).step(flags)
    got = NetRun(_ctx((flag,)), net, B, T).step(flags)
    bad = _diff(ref, got)
    assert not bad[1], f"{case} {flag}: {bad[1]} outputs differ from the default, e.g. {bad[0]}"


def _kernel_key(b):
    ks = lambda L: tuple((k["family"], k["bn"], k["bk"], k["mt"], k["tma_epi"], k["fold"]) for k in L)
    return ks(b["fwd"]), ks(b["dgrad"]), b["wg_form"]


@pytest.mark.parametrize("flag", KERNEL_CHOICE)
def test_switch_tape_parity_generator(flag):
    """Switches that change the kernel of some blocks: the tape parity of the generator's blocks whose kernels change."""
    net, B, T, flags = NET_CASES["generator"]
    ctx = _ctx()
    NetRun(ctx, net, B, T).forward(flags)
    base = {b["name"]: _kernel_key(b) for b in ctx.train_blocks(net)}
    ctx2 = _ctx((flag,))
    NetRun(ctx2, net, B, T).forward(flags)
    changed = [b["name"] for b in ctx2.train_blocks(net) if _kernel_key(b) != base[b["name"]]]
    assert changed, f"{flag} changes no kernel of the generator's training plan"
    _blocks, worst, checked = tape_parity("generator", (flag,), set(changed))
    _report(f"generator {flag} ({len(checked)} blocks)", worst)
    assert len(checked) == len(changed)


@pytest.mark.parametrize("case", ["generator", "syncnet", "disc-input-grad", "disc"])
def test_accumulate_adds_exactly(case):
    """backward(d1) -> G1, backward(d2) -> G2; then backward(d1), backward(d2, ACCUMULATE) == fp32(G1 + G2) bit for bit,
    every bound gradient; the conv bias under a BatchNorm stays exactly 0."""
    net, B, T, flags = NET_CASES[case]
    run = NetRun(_ctx(), net, B, T)
    d1 = run.dout
    g = torch.Generator().manual_seed(77)
    d2 = [torch.randn(d.shape, generator=g).cuda() if d is not None else None for d in d1]
    run.forward(flags | NO_STAT_UPDATE)
    for gr in run.grad.values():
        gr.fill_(float("nan"))
    run.backward(flags, d1)
    g1 = {k: v.clone() for k, v in run.grad.items()}
    run.backward(flags, d2)
    g2 = {k: v.clone() for k, v in run.grad.items()}
    run.backward(flags, d1)
    run.backward(flags | ACCUMULATE, d2)
    bad = [k for k in run.grad if not torch.equal(run.grad[k], g1[k] + g2[k])]
    assert not bad, f"{case}: accumulated gradients differ from G1 + G2 in {len(bad)} tensors, e.g. {bad[:6]}"
    for k, v in run.grad.items():
        assert torch.isfinite(v).all(), k
        if k.endswith("conv_block.0.bias") and net != DISC:
            assert torch.count_nonzero(v) == 0, k


@pytest.mark.parametrize("case", ["generator", "syncnet", "disc"])
def test_no_stat_update_leaves_running_stats(case):
    net, B, T, flags = NET_CASES[case]
    run = NetRun(_ctx(), net, B, T)
    before = run.running()
    run.step(flags | NO_STAT_UPDATE)
    assert all(torch.equal(v, run.val[k]) for k, v in before.items())
    run.step(flags)
    assert sum(not torch.equal(v, run.val[k]) for k, v in before.items()) == len(before)


# ------------------------------------------------------------------------------------------------------------------
# coverage
# ------------------------------------------------------------------------------------------------------------------
def _coverage_items(blocks):
    seen = set()
    for b in blocks:
        s, k = (b["sh"], b["sw"]), (b["kh"], b["kw"])
        if b["has_wgrad"]:
            seen.add(("wgrad BN", b["wg_bn"]))
            form = b["wg_form"]
            seen.add(("form", ["plain", "strided", "transposed", "swap", "folded"][form]))
            if form == 1:
                seen.add(("strided", s))
            if form == 2 and b["h_in"] == 1 and b["w_in"] == 1:
                seen.add(("form", "transposed 1x1 -> 3x3"))
            if form == 4 and b["cin"] == 6:
                seen.add(("form", "folded 7x7 6-channel"))
            if b["wg_ngroups"] > 1 and b["wg_ntaps"] % b["wg_tg"]:
                seen.add(("tap groups", "short last group"))
            if b["wg_m_tiles"] > 1:
                seen.add(("tiles", "m_tiles > 1"))
            if b["wg_n_tiles"] > 1:
                seen.add(("tiles", "n_tiles > 1"))
            sp = b["wg_splits"]
            seen.add(("splits", "1" if sp == 1 else "2-3" if sp <= 3 else ">=4, %4 != 0" if sp % 4 else ">=4, %4 == 0"))
        if b["has_dx"]:
            if b["kind"] == 1:
                f = "strided conv of a convT"
            elif s == (1, 1):
                f = "widened 128" if 64 < -(-b["cin"] // 16) * 16 < 128 and b["cin"] % 64 else "flipped taps"
            else:
                op = b["h_in"] - ((b["h_out"] - 1) * b["sh"] - 2 * b["ph"] + b["kh"])
                f = "transposed phases, out_pad != 0" if op else "transposed phases, out_pad 0"
            seen.add(("dgrad", f))
            if b["has_du"]:
                seen.add(("dgrad", f + " + du"))
            if b["has_dx_add"]:
                seen.add(("dgrad", f + " + dx_add"))
    return seen


REQUIRED = ({("wgrad BN", n) for n in (16, 32, 64, 128)}
            | {("form", f) for f in ("plain", "strided", "transposed", "swap", "folded", "transposed 1x1 -> 3x3",
                                     "folded 7x7 6-channel")}
            | {("strided", s) for s in ((2, 2), (3, 1), (1, 2), (3, 2))}
            | {("tap groups", "short last group"), ("tiles", "m_tiles > 1"), ("tiles", "n_tiles > 1")}
            | {("splits", s) for s in ("1", "2-3", ">=4, %4 != 0", ">=4, %4 == 0")}
            | {("dgrad", f) for f in ("flipped taps", "flipped taps + du", "flipped taps + dx_add",
                                      "transposed phases, out_pad != 0", "transposed phases, out_pad != 0 + dx_add",
                                      "transposed phases, out_pad 0", "strided conv of a convT", "widened 128",
                                      "widened 128 + du")})


def test_coverage():
    """Every item above is reached by a block the tape tests or the block cases checked.  A convT never has a residual
    or skip gradient in these networks (no transposed block is residual or the first block of an encoder stage), and
    the block entry adds neither, so that combination is not required."""
    missing_cases = [c for c in NET_CASES if c not in _BLOCKS] + [c[0] for c in BLOCK_CASES if "block " + c[0] not in _BLOCKS]
    assert not missing_cases, f"run the whole file: these cases did not pass first {missing_cases}"
    seen = set()
    for blocks in _BLOCKS.values():
        seen |= _coverage_items(blocks)
    print("REPORT coverage: " + "; ".join(f"{a}: {b}" for a, b in sorted(seen, key=str)), flush=True)
    missing = REQUIRED - seen
    assert not missing, f"not reached by any checked block: {sorted(missing, key=str)}"
