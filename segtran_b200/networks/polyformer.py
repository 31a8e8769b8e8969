"""Polyformer layer on the H100 kernels (SURVEY.md §8 f.3): the reference's code/networks/polyformer.py:8-106 — a squeezed
attention block WITHOUT the expansion FFN (both CrossAttFeatTrans run multi-mode, their value modes are soft-aggregated,
segtran_shared.py:452-457) applied to a 2x average-pooled CNN feature map and added back to it.

Same classes, constructor signatures and parameter names as the reference (`Polyformer(feat_dim, chan_axis=1, args=None)`,
`polyformer_layers.0.{in_ator_trans,ator_out_trans,attractors}`), so its checkpoints load.  The attention, value
projection, mode aggregation, LayerNorm, bilinear up-sampling and residual run on the library's kernels; the 2x2 average
pooling in front is the stock PyTorch op (it belongs to the CNN side of the block, like the backbone)."""
from __future__ import annotations

import torch
import torch.nn as nn
from torch.nn import Parameter

from .. import ops
from .segtran_shared import CrossAttFeatTrans, SegtranConfig, SegtranInitWeights


# Options a Polyformer takes from the command line (polyformer.py:62-78), with the values used when it is built without args
_ARG_DEFAULTS = (("num_attractors", 256), ("num_modes", 4), ("tie_qk_scheme", "loose"), ("qk_have_bias", True),
                 ("pos_code_type", "lsinu"))


def _polyformer_config(feat_dim, chan_axis, args):
    """SegtranConfig of a one-layer Polyformer: every width equals `feat_dim`, the value projection has no bias, and the
    expansion block only aggregates its value modes (has_FFN = False: no mid / output transformation, polyformer.py:84-87)."""
    cfg = SegtranConfig()
    for key, default in _ARG_DEFAULTS:
        setattr(cfg, key, default if args is None else getattr(args, key))
    if cfg.num_modes == -1:                           # "-1" on the command line means the default number of modes
        cfg.num_modes = 4
    for key in ("in_feat_dim", "feat_dim", "min_feat_dim"):
        setattr(cfg, key, feat_dim)
    for key in ("v_has_bias", "has_FFN", "ablate_multihead", "poly_do_layernorm"):
        setattr(cfg, key, False)
    cfg.num_layers, cfg.chan_axis = 1, chan_axis
    return cfg


class PolyformerLayer(SegtranInitWeights):
    """One squeezed-attention block on a 2x-pooled feature map.  Module / parameter creation order is the reference's
    (in_ator_trans, ator_out_trans, attractors), so a seeded construction yields the same initial weights."""

    def __init__(self, name, config):
        super().__init__(config)
        if config.poly_do_layernorm:
            raise NotImplementedError("segtran_b200: poly_do_layernorm (off in the reference: it costs 1-2 % accuracy, "
                                      "polyformer.py:42-45)")
        self.name = name
        for key in ("chan_axis", "feat_dim", "num_attractors", "qk_have_bias", "poly_do_layernorm"):
            setattr(self, key, getattr(config, key))
        self.in_ator_trans, self.ator_out_trans = (CrossAttFeatTrans(config, "%s-%s" % (name, stage))
                                                   for stage in ("in-squeeze", "squeeze-out"))
        self.attractors = Parameter(torch.randn(1, self.num_attractors, self.feat_dim))
        self.infeat_norm_layer = nn.LayerNorm(self.feat_dim, eps=1e-12, elementwise_affine=False)
        self.pool2x = nn.AvgPool2d(2)
        for fn in (self.init_weights, self.tie_qk, self.add_identity_bias):      # tying follows the initialisation (:31-33)
            self.apply(fn)

    def forward(self, in_feat):
        """in_feat [B,C,H,W] (chan_axis = 1) -> in_feat + upsample(squeezed attention over the 2x-pooled map)."""
        pooled = self.pool2x(in_feat).transpose(self.chan_axis, -1)           # reference :41 swaps C with the LAST dim
        tokens = pooled.reshape(in_feat.shape[0], -1, self.feat_dim).contiguous()
        bank = self.in_ator_trans(self.attractors, tokens)                    # attractors are batch-invariant: batch 1
        fused = self.ator_out_trans(tokens, bank).view(pooled.shape).transpose(self.chan_axis, -1)
        up = ops.resize_linear(fused.contiguous(), tuple(in_feat.shape[2:]))  # bilinear, align_corners=False
        return ops.add(in_feat, up)


class Polyformer(nn.Module):
    def __init__(self, feat_dim, chan_axis=1, args=None):
        super().__init__()
        config = _polyformer_config(feat_dim, chan_axis, args)
        self.polyformer_layers = nn.Sequential(*[PolyformerLayer(str(i), config) for i in range(config.num_layers)])

    def forward(self, in_feat):
        return self.polyformer_layers(in_feat)
