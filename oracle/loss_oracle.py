"""ORACLE (test infrastructure only — used by tests/ and nothing else): the script-level loss functions of the
evaluation loops, restated on torch CPU.  The reference defines them at module level of scripts that parse argv on
import (wav2lip_train.py, color_syncnet_train.py), so they cannot be imported; their arithmetic IS torch's
(nn.BCELoss, F.cosine_similarity, nn.L1Loss), which is what is called here — fp32, CPU.

  cosine_loss      /root/reference/wav2lip_train.py:178-183  (same text in color_syncnet_train.py:133-138, hq_wav2lip_train.py)
  recon_loss       /root/reference/wav2lip_train.py:191
  get_sync_loss    /root/reference/wav2lip_train.py:192-198  (syncnet_T = 5, hparams.py)

Mode of the expert: wav2lip_train.py:187-189 / hq_wav2lip_train.py:189-191 construct the expert SyncNet, freeze its
parameters and never call .eval() on it, so in the scripts its BatchNorm layers run on BATCH statistics (and keep
updating their running averages) even inside eval_model.  This restatement — like the product — evaluates the expert in
eval mode (running statistics), i.e. what the same function computes once the caller has put the expert in eval mode;
batch-statistics BatchNorm belongs to the training row (SURVEY.md section 8 f1) and is not built.
"""
import torch
from torch import nn

from . import w2l_oracle as O

syncnet_T = 5
logloss = nn.BCELoss()
recon_loss = nn.L1Loss()


def cosine_loss(a, v, y):
    d = nn.functional.cosine_similarity(a, v)
    return logloss(d.unsqueeze(1), y)


def stack_lower_halves(g):
    """wav2lip_train.py:193-194: (B,3,T,H,W) -> (B, 3*T, H//2, W)"""
    g = g[:, :, :, g.size(3) // 2:]
    return torch.cat([g[:, :, i] for i in range(syncnet_T)], dim=1)


def get_sync_loss(syncnet_sd, mel, g):
    a, v = O.syncnet_forward(syncnet_sd, mel, stack_lower_halves(g))
    y = torch.ones(g.size(0), 1).float()
    return cosine_loss(a, v, y)


# ----------------------------------------------------------------------------------------------------------------------
# float64 statements of the training tail: the generator head, the embedding normalisation, the discriminator head and
# the loss gradients that seed every backward.  Plain torch float64 with torch's own clamp arithmetic:
#   BCE         -(t * max(log p, -100) + (1 - t) * max(log1p(-p), -100)), mean over n
#   dBCE/dp     (p - t) / max(p (1 - p), 1e-12) / n
#   cosine      (a . v) / (max(|a|, 1e-8) max(|v|, 1e-8))
#   normalize   r / max(|r|, 1e-12); its backward passes no gradient through the norm while the clamp is active
# tests/test_loss_oracle_grads.py pins each against torch.autograd and against torch's fp32 values at every clamp.
# ----------------------------------------------------------------------------------------------------------------------
BCE_LOG_MIN, BCE_DEN_MIN, COS_EPS, NORM_EPS = -100.0, 1e-12, 1e-8, 1e-12


def _d(t):
    return torch.as_tensor(t).double()


def sigmoid64(s):
    return 1.0 / (1.0 + torch.exp(-_d(s)))


def head_forward(y32, w, b, B, T):
    """output_block.1 (1x1, 32 -> 3) + sigmoid on y32 (N,32,H,W), N = T*B (n = t*B + b); g (B,3,T,H,W), or (N,3,H,W) for
    T = 0.  Also returns the logits s in g's layout."""
    y32, w, b = _d(y32), _d(w).reshape(3, 32), _d(b).reshape(3)
    s = torch.einsum("nchw,oc->nohw", y32, w) + b.view(1, 3, 1, 1)
    if T:
        N, _, H, W = s.shape
        s = s.view(T, B, 3, H, W).permute(1, 2, 0, 3, 4)
    return sigmoid64(s), s


def head_backward(y32, w, g, dg, B, T):
    """the head's backward from dL/dg: (dy32 (N,32,H,W), dw (3,32), db (3), and the magnitude sums |dl| f, |dl| of dw, db)"""
    y32, w, g, dg = _d(y32), _d(w).reshape(3, 32), _d(g), _d(dg)
    dl = dg * g * (1.0 - g)
    if T:
        dl = dl.permute(2, 0, 1, 3, 4).reshape(-1, 3, *dl.shape[-2:])   # (B,3,T,H,W) -> (N = T*B, 3, H, W)
    dy32 = torch.einsum("nohw,oc->nchw", dl, w)
    dw = torch.einsum("nohw,nchw->oc", dl, y32)
    db = dl.sum((0, 2, 3))
    return dy32, dw, db, torch.einsum("nohw,nchw->oc", dl.abs(), y32.abs()), dl.abs().sum((0, 2, 3))


def l2norm(r):
    """F.normalize(r, dim=1) of (B, D) rows"""
    r = _d(r)
    return r / r.norm(dim=1, keepdim=True).clamp_min(NORM_EPS)


def l2norm_backward(r, de):
    """dL/dr of F.normalize from dL/de: (de - e (e . de)) / |r| while |r| > 1e-12, de / 1e-12 at the clamp"""
    r, de = _d(r), _d(de)
    n = r.norm(dim=1, keepdim=True)
    e = r / n.clamp_min(NORM_EPS)
    proj = torch.where(n > NORM_EPS, (e * de).sum(1, keepdim=True), torch.zeros_like(n))
    return (de - e * proj) / n.clamp_min(NORM_EPS)


def _cos_norms(a, v):
    """max(|a|, 1e-8), max(|v|, 1e-8) and their product, formed as sqrt(|a|^2 |v|^2) while neither clamps so that a
    cosine of identical rows is exactly 1"""
    saa, svv = (a * a).sum(1, keepdim=True), (v * v).sum(1, keepdim=True)
    na, nv = saa.sqrt().clamp_min(COS_EPS), svv.sqrt().clamp_min(COS_EPS)
    return na, nv, torch.where((na > COS_EPS) & (nv > COS_EPS), (saa * svv).sqrt(), na * nv)


def cosine_similarity(a, v):
    a, v = _d(a), _d(v)
    _, _, nn = _cos_norms(a, v)
    return (a * v).sum(1) / nn.squeeze(1)


def bce_terms(p, t):
    p, t = _d(p), _d(t)
    return -(t * torch.log(p).clamp_min(BCE_LOG_MIN) + (1.0 - t) * torch.log1p(-p).clamp_min(BCE_LOG_MIN))


def bce(p, t):
    """F.binary_cross_entropy(p, t), mean reduction"""
    return bce_terms(p, t).mean()


def bce_grad(p, t, weight=1.0):
    """d(weight * bce(p, t))/dp"""
    p, t = _d(p), _d(t)
    return weight * (p - t) / (p * (1.0 - p)).clamp_min(BCE_DEN_MIN) / p.numel()


def cosine_bce_grad(a, v, y, scale=1.0):
    """scale * BCE(cosine_similarity(a, v), y) (the scripts' cosine_loss, y None: all ones) and its gradients da, dv"""
    a, v = _d(a), _d(v)
    y = torch.ones(a.shape[0], dtype=torch.float64) if y is None else _d(y).reshape(-1)
    na, nv, nn = _cos_norms(a, v)
    d = cosine_similarity(a, v)
    dd = bce_grad(d, y, scale).unsqueeze(1)
    dk = d.unsqueeze(1)
    # dd/da = v / (|a||v|) - d a / |a|^2, written so that it is exactly 0 for identical rows
    return scale * bce(d, y), dd * (v - dk * a * (nv / na)) / nn, dd * (a - dk * v * (na / nv)) / nn, d


def gen_loss_grad(g, gt, l1_scale, dsync=None, ddisc=None):
    """dL/dg (B,3,T,96,96) of the generator steps: l1_scale * sign(g - gt), plus the expert's input gradient dsync
    (B, 3T, 48, 96) at channel 3t + c of the lower half, plus the discriminator's ddisc (T*B, 3, 48, 96) at n = t*B + b"""
    g, gt = _d(g), _d(gt)
    B, _, T, H, W = g.shape
    d = l1_scale * torch.sign(g - gt)
    if dsync is not None:
        d[..., H // 2:, :] += _d(dsync).view(B, T, 3, H // 2, W).permute(0, 2, 1, 3, 4)
    if ddisc is not None:
        d[..., H // 2:, :] += _d(ddisc).view(T, B, 3, H // 2, W).permute(1, 2, 0, 3, 4)
    return d


def disc_head(feat, w, b):
    """binary_pred (512 -> 1) + sigmoid on feat (N, 512): p (N,), and the logit"""
    s = _d(feat) @ _d(w).reshape(-1) + _d(b).reshape(())
    return sigmoid64(s), s


def disc_head_backward(feat, w, p, dp):
    """dfeat (N, 512), dw (512,), db (1,) from dL/dp, through the sigmoid"""
    feat, w, p, dp = _d(feat), _d(w).reshape(-1), _d(p), _d(dp)
    dl = dp * p * (1.0 - p)
    return dl.unsqueeze(1) * w.unsqueeze(0), dl @ feat, dl.sum().reshape(1)


def disc_bce(p_fake, p_real, disc_wt):
    """the hq step's three BCE means [perceptual (0 when disc_wt is 0), real, fake] and their gradients d_perc (scaled by
    disc_wt), d_fake, d_real"""
    one, zero = torch.ones_like(_d(p_fake)), torch.zeros_like(_d(p_fake))
    perc = bce(p_fake, one) if disc_wt > 0 else torch.zeros((), dtype=torch.float64)
    return ([perc, bce(p_real, one), bce(p_fake, zero)],
            bce_grad(p_fake, one, disc_wt), bce_grad(p_fake, zero), bce_grad(p_real, one))


def combine_losses(sync, l1, perc, wt_sync, wt_disc):
    """the steps' total: wt_sync * sync + wt_disc * perceptual + (1 - wt_sync - wt_disc) * l1"""
    return wt_sync * _d(sync) + wt_disc * _d(perc) + (1.0 - wt_sync - wt_disc) * _d(l1)
