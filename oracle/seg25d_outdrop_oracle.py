"""Float64 restatement of the 2.5-D model's out-FPN head with the --outdrop dropout (CPU, checker only).

Reference: segtran25d.py:351-377 (bridge conv + trilinear fused tokens, depth map 'conv' / 'interpolate' / none, out-FPN
dropout) and :464-477 (class conv, trilinear to the input size), on the reference's permuted [B,C,H1,W1,D] volumes.  The
dropout takes an explicit keep mask in the [B,F',D',H1,W1] layout the dropout head hashes (oracle/head_oracle.keep_mask
regenerates the mask a kernel drew).  `forward` is oracle/seg25d_oracle.forward with this head in place of the
un-collapsed one, pinned to the tests/golden/seg25d_outdrop_*.pt fixtures by a CPU test.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import seg25d_oracle as SO
from oracle import segtran_oracle as O


def _conv1x1(x, W, b):
    W = W.reshape(W.shape[0], -1).double()
    y = torch.einsum('oc,bc...->bo...', W, x.double())
    return y if b is None else y + b.double().reshape((1, -1) + (1,) * (x.dim() - 2))


def head_25d(curr, vfeat, grid, Wb, bb, Wc, bc, out_size, Dk, upd, Wu=None, bu=None, keep=None, p=0.0):
    """curr [B*D2, Cf, H1, W1] slice-major (slice b*D2 + d); vfeat [B, N, F] tokens in (h, w, d) order on grid
    (H2, W2, D3); keep [B, F', D', H1, W1] or None -> logits [B, K, H, W, D] in float64."""
    B = vfeat.shape[0]
    H2, W2, D3 = grid
    BD, Cf, H1, W1 = curr.shape
    D2 = BD // B
    vol = curr.double().view(B, D2, Cf, H1, W1).permute(0, 2, 3, 4, 1)                 # [B, Cf, H1, W1, D2]
    vmap = vfeat.double().view(B, H2, W2, D3, -1).permute(0, 4, 1, 2, 3)
    Y = _conv1x1(vol, Wb, bb) + F.interpolate(vmap, size=(H1, W1, D2), mode='trilinear', align_corners=False)
    if Dk > 1 and upd == 'conv':
        Wu5 = Wu.double().reshape(Wu.shape[0], -1, 1, 1, 1)
        Y = SO.depth_map({"out_fpn_upsampleD.weight": Wu5, "out_fpn_upsampleD.bias": bu.double()}, Y, Dk, upd)
    else:
        Y = SO.depth_map({}, Y, Dk, upd)
    if keep is not None:                     # where() keeps only the bool mask for backward (full-size maps are large)
        Y = torch.where(keep.bool().permute(0, 1, 3, 4, 2), Y, torch.zeros((), dtype=Y.dtype, device=Y.device)) / (1.0 - p)
    s = _conv1x1(Y, Wc, bc)
    return F.interpolate(s, size=tuple(out_size), mode='trilinear', align_corners=False)


def out_fpn_pyramid(p, feats: Sequence[Tensor], B: int, out_layers, in_layers, G: int) -> Tensor:
    """The out-FPN pyramid on permuted volumes (segtran25d.py:317-347), returned slice-major [B*D2, Cf, H1, W1]."""
    def vol(t):
        return t.view(B, -1, *t.shape[1:]).permute(0, 2, 3, 4, 1)

    cur = vol(feats[out_layers[0]])
    for layer in out_layers[:-len(in_layers)]:
        up = F.conv3d(cur, p[f"out_fpn{layer}{layer + 1}_conv3d.weight"], p[f"out_fpn{layer}{layer + 1}_conv3d.bias"])
        hi = F.interpolate(vol(feats[layer + 1]), size=up.shape[2:], mode="trilinear", align_corners=False)
        cur = F.group_norm(up + hi, G, p[f"out_gn{layer + 1}b.weight"], p[f"out_gn{layer + 1}b.bias"])
    Bc, C, h, w, D2 = cur.shape
    return cur.permute(0, 4, 1, 2, 3).reshape(Bc * D2, C, h, w)


def forward(p, feats: Sequence[Tensor], mask: Tensor, B: int, out_size: Sequence[int], *, in_layers, out_layers,
            translayer_dims, num_modes, G: int = 8, D_pool_K: int = 2, upd: str = "conv", input_scale=(1., 1., 1.),
            keep=None, drop_p: float = 0.0, **enc_kw) -> Tensor:
    """Segtran25d.forward after the backbone in train mode with --outdrop, the dropout given by `keep` (None: p = 0)."""
    H, W, D = out_size
    feat = SO.in_fpn(p, feats, in_layers, G)
    tok, vmask, grid = SO.pool_tokens(feat, mask, B, D_pool_K)
    H2, W2, D3 = grid
    scales = (H // H2 / input_scale[0], W // W2 / input_scale[1], D // D3 / input_scale[2])
    pos = O.voxels_pos_for_grid(grid, scales, B, tok.dtype, tok.device)
    fused = O.fusion_encoder(p, "voxel_fusion.", tok, pos, vmask.unsqueeze(2), translayer_dims, num_modes, **enc_kw)
    curr = out_fpn_pyramid(p, feats, B, out_layers, in_layers, G)
    Wu, bu = p.get("out_fpn_upsampleD.weight"), p.get("out_fpn_upsampleD.bias")
    return head_25d(curr, fused, grid, p["out_fpn_bridgeconv3d.weight"], p["out_fpn_bridgeconv3d.bias"],
                    p["out_conv3d.weight"], p["out_conv3d.bias"], out_size, D_pool_K, upd, Wu, bu, keep=keep, p=drop_p)


def keep_mask_torch(seed: int, shape, p: float, device) -> Tensor:
    """head_oracle.keep_mask as a bool tensor computed with int64 torch arithmetic on `device` (products of two values
    below 2^32 wrap modulo 2^64, so their low 32 bits are exact): the full-size mask without a numpy pass."""
    from oracle import head_oracle as HO
    M32 = 0xFFFFFFFF
    n = 1
    for s in shape:
        n *= int(s)
    idx = torch.arange(n, device=device, dtype=torch.int64)
    j = idx & 3
    idx4 = idx >> 2
    half = (j >> 1).bool()
    mul = torch.where(half, torch.tensor(0x85EBCA77, device=device), torch.tensor(0x9E3779B1, device=device))
    key = torch.where(half, torch.tensor(int(HO._key(seed, 1)), device=device),
                      torch.tensor(int(HO._key(seed, 0)), device=device))
    a = (((idx4 & M32) * mul) & M32) ^ key
    a ^= ((idx4 >> 32) * 0xC2B2AE3D) & M32
    a ^= a >> 16
    a = (a * 0x7FEB352D) & M32
    a ^= a >> 15
    a = (a * 0x846CA68B) & M32
    a ^= a >> 16
    field = (a >> ((j & 1) * 16)) & 0xFFFF
    return (field >= HO.drop_p16(p)).view(*shape)
