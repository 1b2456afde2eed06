"""DESIGN VALIDATION for the next scope row (training step, SURVEY.md section 8 f1) — test infrastructure only.

The backward pass of one conv.py block written ONLY in terms of the primitives the forward kernels already implement
(a strided/padded conv, a transposed conv as output phases) plus the two new pieces (wgrad as a pixel-contraction GEMM,
the BatchNorm/ReLU/residual elementwise+reduction pass).  tests/test_backward_recipe.py checks every distinct block
geometry of the three networks against torch autograd, so the weight re-packing rules below are the tested recipe the
round-2 kernels follow:

  dgrad of Conv2d(k, stride 1, pad p)      = Conv2d(dz, W', stride 1, pad k-1-p),   W'[ci,co,r,s] = W[co,ci,k-1-r,k-1-s]
  dgrad of Conv2d(k, stride s>1, pad p)    = ConvTranspose2d(dz, W, stride s, pad p, output_padding = size remainder)
                                             (W (Cout,Cin,kh,kw) IS the transposed-conv layout with in=Cout, out=Cin)
  dgrad of ConvTranspose2d(k, s, p, op)    = Conv2d(dz, W_t as (out=Cin_t, in=Cout_t, kh, kw), stride s, pad p)   (no flip)
  wgrad of Conv2d                          dW[co,ci,r,s]   = sum_{n,y,x} dz[n,co,y,x] * xpad[n,ci, y*sy + r, x*sx + s]
  wgrad of ConvTranspose2d                 dW_t[ci,co,r,s] = sum_{n,y,x} x[n,ci,y,x] * dzpad[n,co, y*sy + r', x*sx + s'] (see code)
  BatchNorm (batch statistics) + residual + ReLU backward: the standard two-reduction form.
"""
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from .w2l_oracle import BN_EPS, Row, _pair

# Precision model hook: every tensor-core operand (conv / dgrad / wgrad inputs) passes through Q before the contraction,
# and stored activations through QS.  Identity by default; tests/test_precision_model.py sets bf16 rounding to size the
# gradient-parity tolerances of the training kernels.
Q = lambda t: t      # noqa: E731
QS = lambda t: t     # noqa: E731


def set_precision_model(q=None, qs=None):
    global Q, QS
    Q = q if q is not None else (lambda t: t)
    QS = qs if qs is not None else (lambda t: t)


def conv_dgrad(dz: torch.Tensor, w: torch.Tensor, row: Row, in_hw: Tuple[int, int]) -> torch.Tensor:
    kind, _cin, _cout, k, s, p, op, _res = row
    (kh, kw), (sh, sw), (ph, pw) = _pair(k), _pair(s), _pair(p)
    H, W = in_hw
    if kind == "t":
        # transposed conv forward: z = convT(x, w (Cin,Cout,kh,kw)); its input gradient is a plain strided conv of dz
        return F.conv2d(Q(dz), Q(w), None, stride=(sh, sw), padding=(ph, pw))
    if sh == 1 and sw == 1:
        w2 = w.flip(2, 3).transpose(0, 1).contiguous()                 # (Cin, Cout, kh, kw), taps flipped
        return F.conv2d(Q(dz), Q(w2), None, stride=1, padding=(kh - 1 - ph, kw - 1 - pw))
    # strided conv: the transposed conv with the SAME weight tensor; output_padding recovers the rows/cols the forward
    # conv's floor division dropped
    Ho, Wo = dz.shape[2], dz.shape[3]
    oph = H - ((Ho - 1) * sh - 2 * ph + kh)
    opw = W - ((Wo - 1) * sw - 2 * pw + kw)
    return F.conv_transpose2d(Q(dz), Q(w), None, stride=(sh, sw), padding=(ph, pw), output_padding=(oph, opw))


def conv_wgrad(x: torch.Tensor, dz: torch.Tensor, row: Row) -> torch.Tensor:
    """Per-tap GEMMs with the pixel index as the contraction dimension (what the wgrad kernel does)."""
    kind, cin, cout, k, s, p, op, _res = row
    (kh, kw), (sh, sw), (ph, pw) = _pair(k), _pair(s), _pair(p)
    x, dz = Q(x), Q(dz)
    if kind == "t":
        # z[n,co, y*sh - ph + r, x*sw - pw + s] += x[n,ci,y,x] * w[ci,co,r,s]
        N, _, H, W = x.shape
        Ho, Wo = dz.shape[2], dz.shape[3]
        dzp = F.pad(dz, (pw, pw + sw, ph, ph + sh))                   # index (y*sh + r, x*sw + s) after shifting by the padding
        dw = torch.zeros((cin, cout, kh, kw), dtype=x.dtype)
        xm = x.permute(1, 0, 2, 3).reshape(cin, -1)                   # (Cin, N*H*W)
        for r in range(kh):
            for c in range(kw):
                win = dzp[:, :, r:r + (H - 1) * sh + 1:sh, c:c + (W - 1) * sw + 1:sw]     # (N, Cout, H, W)
                valid = win                                            # out-of-range rows are the zero padding
                dw[:, :, r, c] = xm @ valid.permute(1, 0, 2, 3).reshape(cout, -1).t()
        return dw
    N, _, H, W = x.shape
    Ho, Wo = dz.shape[2], dz.shape[3]
    xp = F.pad(x, (pw, pw, ph, ph))
    dzm = dz.permute(1, 0, 2, 3).reshape(cout, -1)                    # (Cout, N*Ho*Wo)
    dw = torch.zeros((cout, cin, kh, kw), dtype=x.dtype)
    for r in range(kh):
        for c in range(kw):
            win = xp[:, :, r:r + (Ho - 1) * sh + 1:sh, c:c + (Wo - 1) * sw + 1:sw]       # (N, Cin, Ho, Wo)
            dw[:, :, r, c] = dzm @ win.permute(1, 0, 2, 3).reshape(cin, -1).t()
    return dw


def block_forward_train(x, w, b, gamma, beta, row: Row):
    """Forward of one block in train mode, returning what the backward needs (z_hat and invstd instead of z)."""
    kind, _cin, _cout, _k, s, p, op, res = row
    if kind == "t":
        z = F.conv_transpose2d(Q(x), Q(w), b, stride=_pair(s), padding=_pair(p), output_padding=_pair(op))
    else:
        z = F.conv2d(Q(x), Q(w), b, stride=_pair(s), padding=_pair(p))
    if kind == "n":
        y = QS(F.leaky_relu(z, 0.01))
        return y, {"z": QS(z)}
    mean = z.mean(dim=(0, 2, 3))
    var = z.var(dim=(0, 2, 3), unbiased=False)
    invstd = (var + BN_EPS).rsqrt()
    zhat = (z - mean[None, :, None, None]) * invstd[None, :, None, None]
    u = zhat * gamma[None, :, None, None] + beta[None, :, None, None]
    if res:
        u = u + x
    y = QS(F.relu(u))
    return y, {"zhat": QS(zhat), "invstd": invstd, "y": y}


def block_backward(dy, x, w, gamma, row: Row, saved) -> dict:
    """Gradients of one block given dL/dy: dx, dw, db (conv bias), dgamma, dbeta."""
    kind, _cin, _cout, _k, _s, _p, _op, res = row
    if kind == "n":
        z = saved["z"]
        dz = dy * torch.where(z > 0, torch.ones_like(z), torch.full_like(z, 0.01))
        dres = None
        dgamma = dbeta = None
    else:
        du = dy * (saved["y"] > 0).to(dy.dtype)                          # ReLU mask from the stored output
        dres = du if res else None                                       # conv.py:16-18: the skip joins before the ReLU
        zhat, invstd = saved["zhat"], saved["invstd"]
        m = du.numel() / du.shape[1]
        dbeta = du.sum(dim=(0, 2, 3))
        dgamma = (du * zhat).sum(dim=(0, 2, 3))
        dz = (gamma * invstd)[None, :, None, None] * (du - dbeta[None, :, None, None] / m - zhat * dgamma[None, :, None, None] / m)
    dx = conv_dgrad(dz, w, row, (x.shape[2], x.shape[3]))
    if dres is not None:
        dx = dx + dres
    dw = conv_wgrad(x, dz, row)
    db = dz.sum(dim=(0, 2, 3))                                            # == 0 up to rounding when BatchNorm follows
    return {"dx": dx, "dw": dw, "db": db, "dgamma": dgamma, "dbeta": dbeta}


# ----------------------------------------------------------------------------------------------------------------------
# Network level: the generator's training forward/backward as an explicit schedule of block calls — the op list the
# round-2 training plan will replay (forward order, then the reverse with the skip-concat gradient split and the
# residual gradient accumulation made explicit).  Checked against autograd in tests/test_backward_recipe.py.
# ----------------------------------------------------------------------------------------------------------------------
def _blk(sd, prefix):
    return (sd[f"{prefix}.conv_block.0.weight"], sd[f"{prefix}.conv_block.0.bias"],
            sd.get(f"{prefix}.conv_block.1.weight"), sd.get(f"{prefix}.conv_block.1.bias"))


def generator_forward_backward(sd, audio, face, dloss_dout):
    """Wav2Lip.forward in train mode (4-D call) followed by the full backward given dL/d(output).  Returns
    (output, {parameter name: gradient}).  Only block_forward_train / block_backward and tensor slicing are used."""
    from . import w2l_oracle as O
    tape = []                                                  # (prefix, row, input, saved) in forward order

    def run(x, prefix, row):
        w, b, gamma, beta = _blk(sd, prefix)
        y, saved = block_forward_train(x, w, b, gamma, beta, row)
        tape.append((prefix, row, x, saved))
        return y

    a = audio
    for i, row in enumerate(O.GEN_AUDIO_ENCODER):
        a = run(a, f"audio_encoder.{i}", row)
    feats = []
    x = face
    for i, blk in enumerate(O.GEN_FACE_ENCODER):
        for j, row in enumerate(blk):
            x = run(x, f"face_encoder_blocks.{i}.{j}", row)
        feats.append(x)
    x = a
    cat_split = []                                             # channels of the decoder half of every concat
    for i, blk in enumerate(O.GEN_FACE_DECODER):
        for j, row in enumerate(blk):
            x = run(x, f"face_decoder_blocks.{i}.{j}", row)
        cat_split.append(x.shape[1])
        x = torch.cat((x, feats[len(feats) - 1 - i]), dim=1)
    x = run(x, "output_block.0", O.GEN_OUTPUT_BLOCK0)
    hw, hb = sd["output_block.1.weight"], sd["output_block.1.bias"]
    logits = F.conv2d(x, hw, hb)
    out = torch.sigmoid(logits)

    grads = {}
    # head: sigmoid + 1x1 conv
    dlog = dloss_dout * out * (1 - out)
    grads["output_block.1.weight"] = torch.einsum("nohw,nchw->oc", dlog, x)[:, :, None, None]
    grads["output_block.1.bias"] = dlog.sum(dim=(0, 2, 3))
    dx = F.conv2d(dlog, hw.transpose(0, 1).contiguous())       # 1x1 dgrad

    def back(dy):
        prefix, row, xin, saved = tape.pop()
        w, _b, gamma, _beta = _blk(sd, prefix)
        g = block_backward(dy, xin, w, gamma, row, saved)
        grads[f"{prefix}.conv_block.0.weight"] = g["dw"]
        grads[f"{prefix}.conv_block.0.bias"] = g["db"]
        if g["dgamma"] is not None:
            grads[f"{prefix}.conv_block.1.weight"] = g["dgamma"]
            grads[f"{prefix}.conv_block.1.bias"] = g["dbeta"]
        return g["dx"]

    dx = back(dx)                                              # output_block.0
    dfeats = [None] * len(feats)
    for i in reversed(range(len(O.GEN_FACE_DECODER))):
        c = cat_split[i]
        dfeats[len(feats) - 1 - i] = dx[:, c:]                 # the encoder-skip half of the concat (wav2lip.py:108)
        dx = dx[:, :c]
        for _ in O.GEN_FACE_DECODER[i]:
            dx = back(dx)
    da = dx                                                    # gradient of the audio embedding
    dx = None
    for i in reversed(range(len(O.GEN_FACE_ENCODER))):
        d = dfeats[i] if dx is None else dx + dfeats[i]        # stage output feeds the next stage AND a skip connection
        for _ in O.GEN_FACE_ENCODER[i]:
            d = back(d)
        dx = d
    for _ in O.GEN_AUDIO_ENCODER:
        da = back(da)
    assert not tape
    return out, grads
