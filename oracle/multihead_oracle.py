"""CPU restatement of the multi-head ablation (--multihead; reference segtran_ablation.py:93-253 under
segtran_shared.py:478-610, :819-975): SegtranFusionEncoder with --nosqueeze, every layer a CrossAttFeatTrans whose out_trans
is MultiHeadFeatTrans.  Written from the reference's semantics, like oracle/segtran_oracle.py and oracle/posbias_oracle.py,
whose building blocks it reuses; pure PyTorch, any dtype, so float64 gives the fp32 yardstick.  Eval mode (no dropout).
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import posbias_oracle as PO
from oracle import segtran_oracle as O

Params = Dict[str, Tensor]


def multihead_layer(p: Params, pre: str, h: Tensor, num_modes: int, feat_dim: int, *, bias: Optional[Tensor] = None,
                    pos_code_weight: float = 1.0, attn_clip: float = 500.0, trans_output_type: str = "private",
                    stats: Optional[dict] = None) -> Tensor:
    """CrossAttFeatTrans.forward (:553-610) as self-attention over h [B,N,C], then MultiHeadFeatTrans.forward
    (segtran_ablation.py:228-253).  bias: the dense [N,N] positional-bias matrix or None.  stats['max_attn'] gets the
    maximum score of the call, stats['scores'] the kept (conditionally clamped) scores [B,M,N,N]."""
    M = num_modes
    Wq = p[pre + "query.weight"]
    bq = p.get(pre + "query.bias")
    Wk = p.get(pre + "key.weight", Wq)
    bk = p.get(pre + "key.bias", bq)
    B, N, C = h.shape
    d = C // M                                                         # attention_mode_dim (:486)
    q = F.linear(h, Wq, bq).view(B, N, M, d).permute(0, 2, 1, 3)
    k = F.linear(h, Wk, bk).view(B, N, M, d).permute(0, 2, 1, 3)
    s = torch.matmul(q, k.transpose(-1, -2)) / math.sqrt(d)            # :566-567
    smax = float(s.detach().max())
    if stats is not None:
        stats.setdefault("max_attn", []).append(smax)
    if smax > attn_clip:                                               # :578-580
        s = torch.clamp(s, -attn_clip, attn_clip)
    if bias is not None:
        s = s + pos_code_weight * bias                                 # :590-592
    if stats is not None:
        stats.setdefault("scores", []).append(s)                       # :595-596
    probs = torch.softmax(s, dim=-1)                                   # :601
    # ---- MultiHeadFeatTrans.forward(in_key, probs) ----
    Fd = feat_dim
    dh = Fd // M                                                       # feat_dim_onehead (:191)
    v = F.linear(h, p[pre + "out_trans.first_linear.weight"], p[pre + "out_trans.first_linear.bias"])      # :230 [B,N,F]
    v = v.view(B, N, M, dh).permute(0, 2, 1, 3)                        # :232-237 [B,M,N,dh]
    u = torch.matmul(probs, v)                                         # :238
    u = u.permute(0, 2, 1, 3).reshape(B, N, Fd)                        # :239 heads concatenated, channel h*dh+j
    g = O.gelu_erf(F.linear(u, p[pre + "out_trans.intermediate.shared_linear.weight"],
                            p[pre + "out_trans.intermediate.shared_linear.bias"]))               # :93-121, no dropout
    if trans_output_type == "private":                                 # :125-145, the residual is discarded
        y = F.linear(g, p[pre + "out_trans.output.group_linear.weight"][..., 0],
                     p[pre + "out_trans.output.group_linear.bias"])
    else:                                                              # :149-178, the residual is kept
        y = F.linear(g, p[pre + "out_trans.output.shared_linear.weight"], p[pre + "out_trans.output.shared_linear.bias"]) + u
    return O.layer_norm(y, p[pre + "out_trans.output.resout_norm_layer.weight"],
                        p[pre + "out_trans.output.resout_norm_layer.bias"])


def fusion_encoder_multihead(p: Params, pre: str, vfeat: Tensor, voxels_pos: Tensor, vmask: Tensor,
                             translayer_dims: Sequence[int], num_modes: int, *, pos_code_type: str = "lsinu",
                             grid: Sequence[int] = (), pos_bias_radius: int = 7, pos_code_weight: float = 1.0,
                             attn_clip: float = 500.0, trans_output_type: str = "private",
                             collect: Optional[dict] = None) -> Tensor:
    """SegtranFusionEncoder.forward (:907-975) with --nosqueeze --multihead, eval mode.  'lsinu': the code is added to
    the features, with the comb_norm_layers LayerNorm; 'bias' / 'none': no code on the features (:929-940), and 'bias'
    adds the shared bias matrix to every layer's scores."""
    bias = pe = None
    if pos_code_type == "lsinu":
        pe = O.pos_lsinu(voxels_pos.to(vfeat.dtype), p[pre + "pos_code_layer.pos_coder.pos_fc.weight"],
                         p[pre + "pos_code_layer.pos_coder.pos_fc.bias"])
    elif pos_code_type == "bias":
        bias = PO.dense_bias(p[pre + "pos_code_layer.pos_coder.biases"], pos_bias_radius, grid).to(vfeat.dtype)
    elif pos_code_type != "none":
        raise ValueError(pos_code_type)
    x = vfeat
    for i in range(len(translayer_dims) - 1):
        C, Fd = translayer_dims[i], translayer_dims[i + 1]
        h = O.layer_norm(x, p[pre + f"vfeat_norm_layers.{i}.weight"], p[pre + f"vfeat_norm_layers.{i}.bias"])   # :916
        if pe is not None:
            h = O.layer_norm(h + pos_code_weight * pe[:, :, :C])                                                 # :930-934
        h = h * vmask.to(h.dtype)                                                                                # :946
        x = multihead_layer(p, pre + f"translayers.{i}.", h, num_modes, Fd, bias=bias,
                            pos_code_weight=pos_code_weight if bias is not None else 1.0, attn_clip=attn_clip,
                            trans_output_type=trans_output_type, stats=collect)
    return x
