"""Float64 restatement of the segmentation head with the --upd conv and --outdrop options (CPU, checker only).

Reference: segtran3d.py:364-396 (out-FPN tail: bridge conv + upsampled fused tokens, depth upsampling by 'interp',
'conv' + reshape, or 'none', out-FPN dropout) and :488-496 (class conv on the (H,W,D)-permuted map, trilinear to the
input size); segtran2d.py:304-311 and :427-436.  The dropout takes an explicit keep mask in [B,F',D',H1,W1] layout;
drop_keep1 restates the counter-based hash of csrc/sx_common.cuh so a test can regenerate the mask a kernel drew.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

_M32 = np.uint64(0xFFFFFFFF)


def _key(seed: int, w: int) -> np.ndarray:
    z = (int(seed) + (0x68E31DA4A0761D65 if w else 0x9E3779B97F4A7C15)) & ((1 << 64) - 1)
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & ((1 << 64) - 1)
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & ((1 << 64) - 1)
    z ^= z >> 31
    return np.uint64((z ^ (z >> 32)) & 0xFFFFFFFF)


def drop_p16(p: float) -> int:
    v = np.float32(p) * np.float32(65536.0) + np.float32(0.5)
    return 65535 if v >= np.float32(65535.0) else int(v)


def drop_keep1(seed: int, idx: np.ndarray, p: float) -> np.ndarray:
    """keep(idx) of sx::drop_keep1: bool array, idx an array of flat element indices."""
    idx = np.asarray(idx, dtype=np.uint64)
    j = idx & np.uint64(3)
    idx4 = idx >> np.uint64(2)
    half = (j >> np.uint64(1)).astype(bool)
    mul = np.where(half, np.uint64(0x85EBCA77), np.uint64(0x9E3779B1))
    key = np.where(half, _key(seed, 1), _key(seed, 0))
    with np.errstate(over="ignore"):
        a = (((idx4 & _M32) * mul) & _M32) ^ key
        a ^= ((idx4 >> np.uint64(32)) * np.uint64(0xC2B2AE3D)) & _M32
        a ^= a >> np.uint64(16)
        a = (a * np.uint64(0x7FEB352D)) & _M32
        a ^= a >> np.uint64(15)
        a = (a * np.uint64(0x846CA68B)) & _M32
        a ^= a >> np.uint64(16)
    field = (a >> ((j & np.uint64(1)) * np.uint64(16))) & np.uint64(0xFFFF)
    return field >= np.uint64(drop_p16(p))


def keep_mask(seed: int, shape, p: float) -> torch.Tensor:
    """The mask the dropout head draws for an X of `shape` ([B,F',D',H1,W1] or [B,F',H1,W1]), as float64 0/1."""
    n = int(np.prod(shape))
    return torch.from_numpy(drop_keep1(seed, np.arange(n, dtype=np.uint64), p).reshape(shape).astype(np.float64))


def _conv1x1(x, W, b):
    W = W.reshape(W.shape[0], -1).double()
    y = torch.einsum('oc,bc...->bo...', W, x.double())
    return y if b is None else y + b.double().reshape((1, -1) + (1,) * (x.dim() - 2))


def depth_map(Y, Dk, scheme):
    """The out-FPN map after the depth upsampling (segtran3d.py:372-388).  Y [B,C,D1,H1,W1]; for 'conv' Y is already
    out_fpn_upsampleD's output [B,F'*Dk,D1,H1,W1] and is reshaped to [B,F',Dk*D1,H1,W1] (channel f*Dk+j -> depth j*D1+i)."""
    if Dk <= 1 or scheme == 'none':
        return Y
    B, C, D1, H1, W1 = Y.shape
    if scheme == 'conv':
        return Y.reshape(B, C // Dk, Dk, D1, H1, W1).reshape(B, C // Dk, Dk * D1, H1, W1)
    return F.interpolate(Y, size=(D1 * Dk, H1, W1), mode='trilinear', align_corners=False)


def seg_head_3d(curr, vfeat, Wb, bb, Wc, bc, out_size, Dk, scheme, Wu=None, bu=None, keep=None, p=0.0):
    """curr [B,Cf,D1,H1,W1], vfeat [B,F,D2,H2,W2] (the fused tokens as a map) -> logits [B,K,H,W,D] in float64."""
    curr, vfeat = curr.double(), vfeat.double()
    Y = _conv1x1(curr, Wb, bb) + F.interpolate(vfeat, size=curr.shape[2:], mode='trilinear', align_corners=False)
    if scheme == 'conv' and Dk > 1:
        Y = _conv1x1(Y, Wu, bu)
    X = depth_map(Y, Dk, scheme)
    if keep is not None:
        X = X * keep.double() / (1.0 - p)
    X = X.permute(0, 1, 3, 4, 2)
    s = _conv1x1(X, Wc, bc)
    return F.interpolate(s, size=tuple(out_size), mode='trilinear', align_corners=False)


def seg_head_2d(curr, vfeat, Wb, bb, Wc, bc, out_size, keep=None, p=0.0):
    """curr [B,Cf,H1,W1], vfeat [B,F,H2,W2] -> logits [B,K,H,W] in float64; Wb None: identity bridge."""
    curr, vfeat = curr.double(), vfeat.double()
    up = F.interpolate(vfeat, size=curr.shape[2:], mode='bilinear', align_corners=False)
    Y = (_conv1x1(curr, Wb, bb) if Wb is not None else curr) + up
    if keep is not None:
        Y = Y * keep.double() / (1.0 - p)
    s = _conv1x1(Y, Wc, bc)
    return F.interpolate(s, size=tuple(out_size), mode='bilinear', align_corners=False)
