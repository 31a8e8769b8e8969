"""CPU restatement of the mince transformer (reference segtran_shared.py:38-87, :404-447, :612-785, :852-955):
SegtranFusionEncoder with --mince --nosqueeze and pos_code_type 'bias', 'none' or 'lsinu'.  Written from the reference's
semantics, like oracle/segtran_oracle.py and oracle/posbias_oracle.py, whose building blocks it reuses; pure PyTorch, any
dtype, so float64 gives the fp32 yardstick.  Eval mode (no dropout), FFN with the private output, as the drivers build it.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import posbias_oracle as PO
from oracle import segtran_oracle as O

Params = Dict[str, Tensor]


def scale_grids(grid: Sequence[int], scales: Sequence[float]) -> List[tuple]:
    """int(g / scale) cells per axis for every scale (multi_resize_shape, :38-43)."""
    return [tuple(int(g / s) for g in grid) for s in scales]


def channel_bounds(feat_dim: int, props: Sequence[float]) -> List[int]:
    """Boundaries of the scales' channel windows (fracs_to_indices, :68-87): normalised proportions, int() of each share
    but the last, which takes the remaining channels."""
    fr = np.array(props, dtype=float)
    fr = fr / fr.sum()
    idx = [0]
    for f in fr[:-1]:
        idx.append(idx[-1] + int(f * feat_dim))
    idx.append(feat_dim)
    return idx


def resample(x: Tensor, grid: Sequence[int], scale: Optional[float] = None, size: Optional[Sequence[int]] = None) -> Tensor:
    """Token-major [B, M, N, C] on the row-major `grid` -> [B, M, N', C] by F.interpolate (linear / bilinear /
    trilinear, align_corners=False), either with scale_factor = 1/scale or to `size` (resize_flat_features, :45-66)."""
    B, M, N, C = x.shape
    mode = ("linear", "bilinear", "trilinear")[len(grid) - 1]
    y = x.permute(0, 1, 3, 2).reshape(B, M * C, *grid)
    y = F.interpolate(y, size=None if size is None else tuple(size), scale_factor=None if scale is None else 1.0 / scale,
                      mode=mode, align_corners=False)
    return y.reshape(B, M, C, -1).permute(0, 1, 3, 2)


def mince_layer(p: Params, pre: str, h: Tensor, grid: Sequence[int], num_modes: int, feat_dim: int,
                scales: Sequence[float], props: Sequence[float], biases: Optional[Sequence[Optional[Tensor]]] = None, *,
                pos_code_weight: float = 1.0, attn_clip: float = 500.0, stats: Optional[dict] = None) -> Tensor:
    """CrossMinceAttFeatTrans.forward (:704-785) as self-attention, then ExpandedFeatTrans with mince (:404-476).
    biases: per scale, the dense [N_s, N_s] bias matrix or None.  stats['max_attn'] gets one list (per scale) per call."""
    M = num_modes
    B, N, C = h.shape
    d = C // M
    S = len(scales)
    grids = scale_grids(grid, scales)
    q = F.linear(h, p[pre + "query.weight"], p.get(pre + "query.bias")).view(B, N, M, d).permute(0, 2, 1, 3)
    k = F.linear(h, p[pre + "key.weight"], p.get(pre + "key.bias")).view(B, N, M, d).permute(0, 2, 1, 3)
    qk = channel_bounds(d, [1] * S)                                    # (:633-634) equal split of d
    probs, smaxes = [], []
    for s in range(S):
        qs = resample(q[..., qk[s]:qk[s + 1]], grid, scales[s])
        ks = resample(k[..., qk[s]:qk[s + 1]], grid, scales[s])
        sc = torch.matmul(qs, ks.transpose(-1, -2)) / math.sqrt(d)      # (:735-736) the full d
        smax = float(sc.detach().max())
        smaxes.append(smax)
        if smax > attn_clip:                                           # (:747-749) this scale's own decision
            sc = torch.clamp(sc, -attn_clip, attn_clip)
        if biases is not None and biases[s] is not None:
            sc = sc + pos_code_weight * biases[s]                      # (:760-763)
        probs.append(torch.softmax(sc, dim=-1))
    if stats is not None:
        stats.setdefault("max_attn", []).append(smaxes)
    Fd = feat_dim
    v = F.linear(h, p[pre + "out_trans.first_linear.weight"], p.get(pre + "out_trans.first_linear.bias"))
    v = v.view(B, N, M, Fd).permute(0, 2, 1, 3)
    vb = channel_bounds(Fd, props)                                     # (:353-354) --minceprops over F
    us = []
    for s in range(S):
        vs = resample(v[..., vb[s]:vb[s + 1]], grid, scales[s])
        us.append(resample(torch.matmul(probs[s], vs), grids[s], size=grid))     # (:436-439)
    u = torch.cat(us, dim=-1)                                          # (:443) [B,M,N,F]
    g = O.gelu_erf(F.linear(u, p[pre + "out_trans.intermediate.shared_linear.weight"],
                            p[pre + "out_trans.intermediate.shared_linear.bias"]))
    Wo = p[pre + "out_trans.output.group_linear.weight"].view(M, Fd, Fd)
    bo = p[pre + "out_trans.output.group_linear.bias"].view(M, 1, Fd)
    y = O.layer_norm(torch.einsum("bmnf,mof->bmno", g, Wo) + bo, p[pre + "out_trans.output.resout_norm_layer.weight"],
                     p[pre + "out_trans.output.resout_norm_layer.bias"])
    w = torch.softmax(F.linear(y, p[pre + "out_trans.feat_softaggr.feat2score.weight"],
                               p[pre + "out_trans.feat_softaggr.feat2score.bias"]), dim=1)
    return (y * w).sum(dim=1)


def fusion_encoder_mince(p: Params, pre: str, vfeat: Tensor, voxels_pos: Tensor, vmask: Tensor,
                         translayer_dims: Sequence[int], num_modes: int, pos_code_type: str, grid: Sequence[int],
                         scales: Sequence[float], props: Sequence[float], *, pos_bias_radius: int = 7,
                         pos_code_weight: float = 1.0, attn_clip: float = 500.0, collect: Optional[dict] = None) -> Tensor:
    """SegtranFusionEncoder.forward (:907-955) with --mince --nosqueeze, eval mode.  'bias': one table per scale
    (pos_code_layers.{s}), over that scale's grid, added to its scores; 'none': no positional code; 'lsinu': the single
    learned code added to the features (with the comb_norm_layers LayerNorm), as without mince."""
    grids = scale_grids(grid, scales)
    biases = None
    if pos_code_type == "bias":
        biases = [PO.dense_bias(p[pre + f"pos_code_layers.{s}.pos_coder.biases"], pos_bias_radius, grids[s]).to(vfeat.dtype)
                  for s in range(len(scales))]
    elif pos_code_type == "lsinu":
        pe = O.pos_lsinu(voxels_pos.to(vfeat.dtype), p[pre + "pos_code_layer.pos_coder.pos_fc.weight"],
                         p[pre + "pos_code_layer.pos_coder.pos_fc.bias"])
    elif pos_code_type != "none":
        raise ValueError(pos_code_type)
    x = vfeat
    for i in range(len(translayer_dims) - 1):
        C, Fd = translayer_dims[i], translayer_dims[i + 1]
        h = O.layer_norm(x, p[pre + f"vfeat_norm_layers.{i}.weight"], p[pre + f"vfeat_norm_layers.{i}.bias"])   # :916
        if pos_code_type == "lsinu":
            h = O.layer_norm(h + pos_code_weight * pe[:, :, :C])                                                  # :930-934
        h = h * vmask.to(h.dtype)                                                                                # :946
        x = mince_layer(p, pre + f"translayers.{i}.", h, grid, num_modes, Fd, scales, props, biases,
                        pos_code_weight=pos_code_weight if pos_code_type == "bias" else 1.0, attn_clip=attn_clip,
                        stats=collect)
    return x
