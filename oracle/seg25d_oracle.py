"""Plain-PyTorch restatement of the reference Segtran25d forward minus the backbone (code/networks/segtran25d.py:258-477),
with the reference's layout: the depth pooling and the out-FPN on permuted [B,C,H,W,D] volumes, 3-D GroupNorm, and the
un-collapsed head (bridge conv of the full out-FPN map, depth upsampling, class conv, trilinear).

TEST INFRASTRUCTURE ONLY: pinned to the tests/golden/seg25d_*.pt fixtures (built from the real reference) by a CPU test,
and used as the eager reference formulation by the full-size GPU test and tools/time_segtran25d.py.  The encoder is
oracle.segtran_oracle.fusion_encoder (learnable-sinusoid positions).
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import segtran_oracle as O

Params = Dict[str, Tensor]


def get_mask(batch: Tensor, pool_stride: int) -> Tensor:
    """[B,C',H,W,D] input after in_bridge_to3 -> per-slice nonzero mask [B*D, H/s, W/s] (segtran25d.py:256-262, :405-411)."""
    C = batch.shape[1]
    fake2d = batch.permute(0, 4, 1, 2, 3).reshape(-1, C, *batch.shape[2:4])
    return (F.avg_pool2d(fake2d.abs(), pool_stride).sum(dim=1) > 0).long()


def in_fpn(p: Params, feats: Sequence[Tensor], in_layers: Sequence[int], G: int) -> Tensor:
    """Per-slice 2-D in-FPN ('AN') + bridge conv (segtran25d.py:264-288) -> [B*D2, C0, H2, W2]."""
    cur = feats[in_layers[0]]
    for layer in in_layers[:-1]:
        up = F.conv2d(cur, p[f"in_fpn{layer}{layer + 1}_conv.weight"], p[f"in_fpn{layer}{layer + 1}_conv.bias"])
        hi = F.interpolate(feats[layer + 1], size=up.shape[2:], mode="bilinear", align_corners=False)
        cur = F.group_norm(up + hi, G, p[f"in_gn{layer + 1}b.weight"], p[f"in_gn{layer + 1}b.bias"])
    if "in_fpn_bridgeconv.weight" in p:
        cur = F.conv2d(cur, p["in_fpn_bridgeconv.weight"], p["in_fpn_bridgeconv.bias"])
    return cur


def pool_tokens(feat: Tensor, mask: Tensor, B: int, D_pool_K: int):
    """Depth pooling and flatten (segtran25d.py:290-315): feat [B*D2, C0, H2, W2], mask [B*D2, H2, W2] ->
    tokens [B, H2*W2*D3, C0] in (h, w, d) order, vmask [B, N], grid (H2, W2, D3)."""
    BD, C0, H2, W2 = feat.shape
    D2 = BD // B
    chwd = feat.view(B, D2, C0, H2, W2).permute(0, 2, 3, 4, 1)
    D3 = D2 // D_pool_K
    chwd2 = F.interpolate(chwd, size=(H2, W2, D3), mode="trilinear", align_corners=False)
    m = F.interpolate(mask.view(B, D2, H2, W2).permute(0, 2, 3, 1).float(), size=(W2, D3), mode="bilinear",
                      align_corners=False)
    vmask = (m >= 0.5).long().reshape(B, -1)
    return chwd2.permute(0, 2, 3, 4, 1).reshape(B, -1, C0), vmask, (H2, W2, D3)


def out_fpn(p: Params, feats: Sequence[Tensor], fused_vol: Tensor, B: int, out_layers: Sequence[int],
            in_layers: Sequence[int], G: int, D_pool_K: int, upd: str) -> Tensor:
    """Out-FPN on permuted volumes with 3-D GroupNorm, bridge conv + trilinear tokens, depth map
    (segtran25d.py:317-377) -> the full map [B, F', H1, W1, D']."""
    def vol(t):
        return t.view(B, -1, *t.shape[1:]).permute(0, 2, 3, 4, 1)

    cur = vol(feats[out_layers[0]])
    for layer in out_layers[:-len(in_layers)]:
        up = F.conv3d(cur, p[f"out_fpn{layer}{layer + 1}_conv3d.weight"], p[f"out_fpn{layer}{layer + 1}_conv3d.bias"])
        hi = F.interpolate(vol(feats[layer + 1]), size=up.shape[2:], mode="trilinear", align_corners=False)
        cur = F.group_norm(up + hi, G, p[f"out_gn{layer + 1}b.weight"], p[f"out_gn{layer + 1}b.bias"])
    x = F.conv3d(cur, p["out_fpn_bridgeconv3d.weight"], p["out_fpn_bridgeconv3d.bias"]) + \
        F.interpolate(fused_vol, size=cur.shape[2:], mode="trilinear", align_corners=False)
    return depth_map(p, x, D_pool_K, upd)


def depth_map(p: Params, x: Tensor, D_pool_K: int, upd: str) -> Tensor:
    """Depth upsampling of the out-FPN map [B, F, H1, W1, D2] (segtran25d.py:355-371): 'conv' puts channel f*Dk + j of
    out_fpn_upsampleD at slice i at depth i*Dk + j; 'interpolate' is trilinear x Dk; anything else leaves it."""
    if D_pool_K > 1 and upd == "conv":
        y = F.conv3d(x, p["out_fpn_upsampleD.weight"], p["out_fpn_upsampleD.bias"])
        y = y.view((x.shape[0], y.shape[1] // D_pool_K, D_pool_K) + tuple(x.shape[2:])).permute(0, 1, 3, 4, 5, 2)
        return y.reshape(tuple(y.shape[:4]) + (-1,))
    if D_pool_K > 1 and upd == "interpolate":
        return F.interpolate(x, size=(x.shape[2], x.shape[3], x.shape[4] * D_pool_K), mode="trilinear",
                             align_corners=False)
    return x


def forward(p: Params, feats: Sequence[Tensor], mask: Tensor, B: int, out_size: Sequence[int], *,
            in_layers: Sequence[int], out_layers: Sequence[int], translayer_dims: Sequence[int], num_modes: int,
            G: int = 8, D_pool_K: int = 2, upd: str = "conv", input_scale=(1., 1., 1.), **enc_kw) -> Tensor:
    """Segtran25d.forward after the backbone: feats = the backbone's five per-slice maps [B*D2, C_l, h_l, w_l],
    mask [B*D2, H2, W2] (get_mask), out_size = (H, W, D) -> logits [B, K, H, W, D].  Parameter names as in
    Segtran25d.state_dict()."""
    H, W, D = out_size
    feat = in_fpn(p, feats, in_layers, G)
    tok, vmask, grid = pool_tokens(feat, mask, B, D_pool_K)
    H2, W2, D3 = grid
    scales = (H // H2 / input_scale[0], W // W2 / input_scale[1], D // D3 / input_scale[2])
    pos = O.voxels_pos_for_grid(grid, scales, B, tok.dtype, tok.device)
    fused = O.fusion_encoder(p, "voxel_fusion.", tok, pos, vmask.unsqueeze(2), translayer_dims, num_modes, **enc_kw)
    fused_vol = fused.view(B, H2, W2, D3, -1).permute(0, 4, 1, 2, 3)
    if list(out_layers) != list(in_layers):
        x = out_fpn(p, feats, fused_vol, B, out_layers, in_layers, G, D_pool_K, upd)
        s = F.conv3d(x, p["out_conv3d.weight"], p["out_conv3d.bias"])
    else:
        s = F.conv_transpose3d(fused_vol, p["out_conv3d.weight"], p["out_conv3d.bias"], stride=(2, 2, 1))
    return F.interpolate(s, size=tuple(out_size), mode="trilinear", align_corners=False)
