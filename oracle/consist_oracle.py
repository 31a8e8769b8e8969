"""Plain-PyTorch (CPU, any dtype) restatement of the attention-consistency losses of the reference training drivers:
train3d.py:426-449 (BCE-with-logits against the class-consistency matrix) and train2d.py:668-723 (margin rule around the
per-batch mean, capped at 1).  TEST INFRASTRUCTURE ONLY: the checker of segtran_b200.train.attn_consist_loss3d/2d.

It forms the [B,N,N] matrices the CUDA path avoids, so it is meant for small shapes."""
from __future__ import annotations

import torch
import torch.nn.functional as F


def flat_mask(mask, orig_feat_shape, three_d):
    """The reference's mask preparation: (3-D) [B,C,H,W,D] -> [B,C,D,H,W], then trilinear / bilinear resize
    (align_corners=False) to orig_feat_shape, flattened to [B,C,N]."""
    if three_d:
        mask = mask.permute(0, 1, 4, 2, 3)
    r = F.interpolate(mask, size=tuple(orig_feat_shape), mode='trilinear' if three_d else 'bilinear', align_corners=False)
    return r.reshape(r.shape[0], r.shape[1], -1)


def affinity(entry):
    """[in_ator [B,1,A,N], ator_out [B,1,N,A]] -> ator_out @ in_ator; a dense [B,1,N,N] entry as it is; -> [B,N,N]."""
    if isinstance(entry, (list, tuple)):
        xi, xo = entry
        entry = torch.matmul(xo, xi)
    return entry.squeeze(1)


def targets(fm):
    return torch.clip(torch.matmul(fm.transpose(-2, -1), fm), 0, 1)


def layer_bce(x, c):
    return F.binary_cross_entropy_with_logits(x, c)


def layer_margin(x, c):
    mu = x.mean(dim=2, keepdim=True).mean(dim=1, keepdim=True)
    cb = c.bool()
    inc = ((x < mu) & cb) | ((x > mu - 0.1) & ~cb)
    return (x - mu)[inc].abs().mean()


def consist_loss3d(layers_attn_scores, orig_feat_shape, mask, only_first_layer=True):
    c = targets(flat_mask(mask, orig_feat_shape, True))
    n = 1 if only_first_layer else len(layers_attn_scores)
    loss = 0
    for e in layers_attn_scores[:n]:
        loss = loss + layer_bce(affinity(e), c)
    return loss / n


def consist_loss2d(layers_attn_scores, orig_feat_shape, mask, only_first_layer=False):
    c = targets(flat_mask(mask, orig_feat_shape, False))
    n = 1 if only_first_layer else len(layers_attn_scores)
    loss = 0
    for e in layers_attn_scores[:n]:
        loss = loss + layer_margin(affinity(e), c)
    loss = loss / n
    if loss > 1:
        loss = loss / loss.item()
    return loss
