"""CPU restatement of the positional-code ablations of SegtranFusionEncoder (reference segtran_shared.py:819-975,
:1002-1238): pos_code_type 'bias' (sliding-window biases added to the attention scores of the plain --nosqueeze
attention) and 'none' (no positional code).  Written from the reference's semantics, like oracle/segtran_oracle.py,
whose building blocks it reuses; pure PyTorch, any dtype, so float64 gives the fp32 yardstick.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import segtran_oracle as O

Params = Dict[str, Tensor]


def dense_bias(table: Tensor, R: int, grid: Sequence[int]) -> Tensor:
    """The [N,N] matrix SlidingPosBiases2D/3D.forward builds: bias[q,k] = table[k - q + R] (per dimension) when every
    |k_i - q_i| <= R, else 0; tokens are the row-major cells of `grid`."""
    c = O.gen_all_indices(grid).reshape(-1, len(grid))
    diff = c[None, :, :] - c[:, None, :]                      # k - q   [q, k, pd]
    inwin = (diff.abs() <= R).all(-1)
    idx = (diff + R).clamp(0, 2 * R)
    vals = table[tuple(idx[..., i] for i in range(len(grid)))]
    return torch.where(inwin, vals, torch.zeros((), dtype=table.dtype))


def cross_att_biased(p: Params, pre: str, h: Tensor, num_modes: int, feat_dim: int, bias: Tensor, *,
                     pos_code_weight: float = 1.0, attn_clip: float = 500.0, stats: Optional[dict] = None) -> Tensor:
    """CrossAttFeatTrans.forward (:553-610) as self-attention with pos_biases: the clamp is decided on the raw scores,
    then S' = clamp_if(S) + pos_code_weight * bias, softmax; then ExpandedFeatTrans with the FFN and the private output
    (:404-476).  Eval mode (no dropout)."""
    M = num_modes
    Wq = p[pre + "query.weight"]
    bq = p.get(pre + "query.bias")
    Wk = p.get(pre + "key.weight", Wq)
    bk = p.get(pre + "key.bias", bq)
    B, N, C = h.shape
    d = C // M
    q = F.linear(h, Wq, bq).view(B, N, M, d).permute(0, 2, 1, 3)
    k = F.linear(h, Wk, bk).view(B, N, M, d).permute(0, 2, 1, 3)
    s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(d)            # :566-567
    smax = float(s.detach().max())
    if stats is not None:
        stats.setdefault("max_attn", []).append(smax)
    if smax > attn_clip:                                               # :578-580
        s = torch.clamp(s, -attn_clip, attn_clip)
    s = s + pos_code_weight * bias                                     # :590-592
    probs = torch.softmax(s, dim=-1)                                   # :601
    Fd = feat_dim
    v = F.linear(h, p[pre + "out_trans.first_linear.weight"], p.get(pre + "out_trans.first_linear.bias"))
    u = torch.matmul(probs, v.view(B, N, M, Fd).permute(0, 2, 1, 3))   # :447
    g = O.gelu_erf(F.linear(u, p[pre + "out_trans.intermediate.shared_linear.weight"],
                            p[pre + "out_trans.intermediate.shared_linear.bias"]))
    Wo = p[pre + "out_trans.output.group_linear.weight"].view(M, Fd, Fd)
    bo = p[pre + "out_trans.output.group_linear.bias"].view(M, 1, Fd)
    y = O.layer_norm(torch.einsum("bmnf,mof->bmno", g, Wo) + bo, p[pre + "out_trans.output.resout_norm_layer.weight"],
                     p[pre + "out_trans.output.resout_norm_layer.bias"])
    w = torch.softmax(F.linear(y, p[pre + "out_trans.feat_softaggr.feat2score.weight"],
                               p[pre + "out_trans.feat_softaggr.feat2score.bias"]), dim=1)
    return (y * w).sum(dim=1)


def fusion_encoder_pos(p: Params, pre: str, vfeat: Tensor, vmask: Tensor, translayer_dims: Sequence[int],
                       num_modes: int, pos_code_type: str, *, grid: Sequence[int] = (), pos_bias_radius: int = 7,
                       pos_code_weight: float = 1.0, attn_clip: float = 500.0, use_squeezed_transformer: bool = False,
                       collect: Optional[dict] = None) -> Tensor:
    """SegtranFusionEncoder.forward (:907-975), eval mode, pos_code_type 'bias' (plain attention) or 'none' (either):
    h = LN_{g,b}(x) * mask — no positional code and no comb_norm_layers LayerNorm (:929-940) — then the layer, which gets
    the shared bias matrix in 'bias' mode (:947-955)."""
    if pos_code_type not in ("bias", "none"):
        raise ValueError(pos_code_type)
    if pos_code_type == "bias" and use_squeezed_transformer:
        raise ValueError("positional biases need the plain transformer (reference :841-844)")
    bias = None
    if pos_code_type == "bias":
        bias = dense_bias(p[pre + "pos_code_layer.pos_coder.biases"], pos_bias_radius, grid).to(vfeat.dtype)
    x = vfeat
    for i in range(len(translayer_dims) - 1):
        Fd = translayer_dims[i + 1]
        h = O.layer_norm(x, p[pre + f"vfeat_norm_layers.{i}.weight"], p[pre + f"vfeat_norm_layers.{i}.bias"])   # :916
        h = h * vmask.to(h.dtype)                                                                                # :946
        lp = pre + f"translayers.{i}."
        if bias is not None:
            x = cross_att_biased(p, lp, h, num_modes, Fd, bias, pos_code_weight=pos_code_weight, attn_clip=attn_clip,
                                 stats=collect)
        elif use_squeezed_transformer:
            x = O.squeezed_layer(p, lp, h, num_modes, Fd, attn_clip=attn_clip, stats=collect)
        else:
            x = O.cross_att(p, lp, h, h, num_modes, Fd, True, attn_clip=attn_clip, stats=collect)
    return x
