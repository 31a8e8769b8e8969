"""H100-native Squeeze-and-Expansion transformer stack — drop-in module surface.

Mirrors the nn.Module contract of the reference's ``code/networks/segtran_shared.py`` (class names,
constructor signatures, sub-module / parameter names and creation order, so that
``torch.manual_seed(s)`` + construction gives the reference's initial weights and reference
checkpoints load with ``load_state_dict``), while every forward runs on the sm_90a kernels in
``segtran_b200/csrc`` through ``segtran_b200.ops``.  There is no PyTorch fallback inside the stack.

Supported configuration = the one the reference's drivers force (train3d.py:174-178, train2d.py:245-249):
squeezed attention (or plain cross attention), pos_code_type 'lsinu', mid_type 'shared',
trans_output_type 'private'|'shared', tie_qk 'shared'|'loose'|'none', pool_modes_feat 'softmax', plus
--nosqueeze and --squeezeuseffn, the positional-code ablations --pos bias (sliding-window biases inside the
attention softmax, plain attention only) and --pos none, the mince transformer (--mince with --nosqueeze: plain
attention on several downsampled copies of the token grid) and the multi-head ablation (--multihead with --nosqueeze:
MultiHeadFeatTrans).  The other ablation-only switches (rand/sinu position codes, mid_type 'private') raise
NotImplementedError.
"""
from __future__ import annotations

import copy
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops

# backbone name -> channel widths of its five feature maps (reference: segtran_shared.py:15-26)
bb2feat_dims = {
    'resnet34': [64, 64, 128, 256, 512], 'resnet50': [64, 256, 512, 1024, 2048],
    'resnet101': [64, 256, 512, 1024, 2048], 'resibn101': [64, 256, 512, 1024, 2048],
    'eff-b0': [16, 24, 40, 112, 1280], 'eff-b1': [16, 24, 40, 112, 1280], 'eff-b2': [16, 24, 48, 120, 1408],
    'eff-b3': [24, 32, 48, 136, 1536], 'eff-b4': [24, 32, 56, 160, 1792], 'effv2m': [24, 48, 80, 176, 512],
    'i3d': [64, 192, 480, 832, 1024],
}


def gen_all_indices(shape, device):
    """Coordinates of every cell of a grid, [*shape, len(shape)] (reference segtran_shared.py:28-36)."""
    axes = [torch.arange(int(s), device=device) for s in shape]
    return torch.stack(torch.meshgrid(*axes, indexing='ij'), dim=len(axes))


def multi_resize_shape(shape, scales):
    """The token grid of every mince scale: int(g / scale) cells per axis (reference segtran_shared.py:38-43)."""
    return [torch.Size([int(g / scale) for g in shape]) for scale in scales]


def mince_grids(shape, scales):
    """multi_resize_shape, checked against what F.interpolate(scale_factor=1/scale) produces (floor(g * (1/scale)) cells,
    which the reference's reshapes rely on): a scale that empties an axis or where the two disagree raises ValueError."""
    grid = tuple(int(g) for g in shape)
    if len(grid) not in (2, 3):
        raise ValueError("mince transformer: a 2-D or 3-D token grid is needed (got %s)" % (grid,))
    out = []
    for scale, shp in zip(scales, multi_resize_shape(grid, scales)):
        for g, n in zip(grid, shp):
            if n < 1:
                raise ValueError("mince transformer: scale %s leaves an empty axis of the grid %s" % (scale, grid))
            if n != math.floor(g * (1.0 / scale)):
                raise ValueError("mince transformer: scale %s gives int(%d / %s) = %d cells but F.interpolate makes %d"
                                 % (scale, g, scale, n, math.floor(g * (1.0 / scale))))
        out.append(tuple(int(n) for n in shp))
    return out


def fracs_to_indices(feat_dim, mince_channel_props):
    """Channel boundaries of the mince scales (reference segtran_shared.py:68-87): the proportions (fractions or
    unnormalised weights) are normalised; scale i < last gets int(frac_i * feat_dim) channels, the last one the rest.
    -> (boundaries [S+1], widths [S])."""
    fracs = np.array(mince_channel_props, dtype=float)
    fracs /= fracs.sum()
    n = len(fracs)
    idx = [0] * (n + 1)
    for i in range(n - 1):
        idx[i + 1] = idx[i] + int(fracs[i] * feat_dim)
    idx[-1] = feat_dim
    return idx, [idx[i + 1] - idx[i] for i in range(n)]


def _check_mince_config(config):
    if config.mince_scales is None or config.mince_channel_props is None:
        raise ValueError("mince transformer: mince_scales and mince_channel_props must be given")
    if len(config.mince_channel_props) != len(config.mince_scales):
        raise ValueError("mince transformer: %d scales but %d channel proportions"
                         % (len(config.mince_scales), len(config.mince_channel_props)))




class SegtranConfig:
    """Application-independent settings (reference segtran_shared.py:90-196); same attribute names and defaults."""

    def __init__(self):
        self.feat_dim = -1
        self.in_feat_dim = -1
        self.num_modes = 4
        self.use_squeezed_transformer = True
        self.num_attractors = 256
        self.tie_qk_scheme = 'shared'
        self.mid_type = 'shared'
        self.trans_output_type = 'private'
        self.act_fun = F.gelu
        self.has_FFN = True
        self.has_FFN_in_squeeze = False
        self.pos_code_type = 'lsinu'
        self.pos_code_weight = 1.
        self.pos_bias_radius = 7
        self.qk_have_bias = True
        self.v_has_bias = False
        self.attn_clip = 500
        self.base_initializer_range = 0.02
        self.query_idbias_scale = 10
        self.feattrans_lin1_idbias_scale = 10
        self.pool_modes_feat = 'softmax'
        self.use_mince_transformer = False
        self.mince_scales = None
        self.mince_channel_props = None
        self.hidden_dropout_prob = 0.1
        self.attention_probs_dropout_prob = 0.1
        self.out_fpn_do_dropout = False
        self.eval_robustness = False
        self.ablate_multihead = False
        self.use_attn_consist_loss = False

    def try_assign(self, args, *keys):
        hit = False
        for key in keys:
            if key in args:
                self.__dict__[key] = args[key] if isinstance(args, dict) else args.__dict__[key]
                hit = True
        return hit

    def set_fpn_layers(self, config_name, fpn_settings, do_print=True):
        self.in_fpn_layers = [int(c) for c in fpn_settings.in_fpn_layers]
        self.out_fpn_layers = [int(c) for c in fpn_settings.out_fpn_layers]
        if self.out_fpn_layers[-1] > self.in_fpn_layers[-1]:
            print("in_fpn_layers=%s is not compatible with out_fpn_layers=%s" % (self.in_fpn_layers, self.out_fpn_layers))
            exit(0)
        ratios = fpn_settings.translayer_compress_ratios
        assert len(ratios) == self.num_translayers + 1, \
            "Length of {} != 1 + num_translayers {}".format(ratios, self.num_translayers)
        self.orig_in_feat_dim = self.bb_feat_dims[self.in_fpn_layers[-1]]
        self.translayer_compress_ratios = ratios
        self.translayer_dims = [int(self.orig_in_feat_dim / r) for r in np.cumprod(ratios)]
        self.trans_in_dim = self.translayer_dims[0]
        self.min_feat_dim = np.min(self.translayer_dims)
        self.trans_out_dim = self.translayer_dims[-1]
        self.in_fpn_scheme = fpn_settings.in_fpn_scheme
        self.out_fpn_scheme = fpn_settings.out_fpn_scheme
        if do_print:
            print("'%s' orig in-feat: %d, in-feat: %d, out-feat: %d, in-scheme: %s, out-scheme: %s, translayer_dims: %s"
                  % (config_name, self.orig_in_feat_dim, self.trans_in_dim, self.trans_out_dim, self.in_fpn_scheme,
                     self.out_fpn_scheme, self.translayer_dims))


def _prod(shape):
    n = 1
    for g in shape:
        n *= int(g)
    return n


def _unsupported(what):
    raise NotImplementedError("segtran_b200: %s is an ablation path this build does not implement "
                              "(use the reference module for it)" % what)


# ---------------------------------------------------------------------------------------------------
# expansion block pieces: parameter holders with the reference's names; the math lives in ExpandedFeatTrans
# ---------------------------------------------------------------------------------------------------
class MMSharedMid(nn.Module):
    """One Linear(F->F) shared by all modes + erf-GELU + dropout (reference :220-251)."""

    def __init__(self, config):
        super().__init__()
        self.num_modes, self.feat_dim = config.num_modes, config.feat_dim
        self.shared_linear = nn.Linear(self.feat_dim, self.feat_dim)
        self.mid_act_fn = config.act_fun
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, x):                       # x [B,M,U,F]
        p = self.dropout.p if self.training else 0.0
        return ops.linear(x, self.shared_linear.weight, self.shared_linear.bias, gelu=True, drop_p=p,
                          seed=ops.new_dropout_seed(x.device) if p > 0 else 0)


class MMPrivateMid(nn.Module):
    def __init__(self, config):
        super().__init__()
        _unsupported("mid_type='private'")


class MMPrivateOutput(nn.Module):
    """Per-mode Linear (grouped 1x1 Conv1d) + dropout + LayerNorm; the reference computes a residual and then
    discards it (:269-272) — reproduced: no shortcut."""

    def __init__(self, config):
        super().__init__()
        self.num_modes, self.feat_dim = config.num_modes, config.feat_dim
        fam = self.feat_dim * self.num_modes
        self.group_linear = nn.Conv1d(fam, fam, 1, groups=self.num_modes)
        self.resout_norm_layer = nn.LayerNorm(self.feat_dim, eps=1e-12, elementwise_affine=True)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, x, shortcut=None):        # x [B,M,U,F] -> un-normalised per-mode projection
        return ops.group_linear(x, self.group_linear.weight, self.group_linear.bias)


class MMSharedOutput(nn.Module):
    """One Linear(F->F) shared by all modes + residual + dropout + LayerNorm (reference :279-308); here the residual
    IS kept (:305), unlike MMPrivateOutput."""

    def __init__(self, config):
        super().__init__()
        self.num_modes, self.feat_dim = config.num_modes, config.feat_dim
        self.shared_linear = nn.Linear(self.feat_dim, self.feat_dim)
        self.resout_norm_layer = nn.LayerNorm(self.feat_dim, eps=1e-12, elementwise_affine=True)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, x, shortcut):             # x, shortcut [B,M,U,F] -> un-normalised sum
        return ops.add(ops.linear(x, self.shared_linear.weight, self.shared_linear.bias), shortcut)


class LearnedSoftAggregate(nn.Module):
    """Linear(F->1) score per mode, softmax over modes, weighted sum (reference :311-325)."""

    def __init__(self, num_feat, group_dim, keepdim=False):
        super().__init__()
        self.group_dim = group_dim
        self.feat2score = nn.Linear(num_feat, 1)
        self.keepdim = keepdim

    def forward(self, x, score_basis=None):
        """x [B,M,U,F] -> [B,U,F] (reference :318-325, group_dim = 1).  The fused LayerNorm + aggregate of the FFN branch
        (ops.ln_softaggr) does not go through here; this is the stand-alone form (no-FFN branch, Polyformer)."""
        if score_basis is not None or self.group_dim != 1 or x.dim() != 4:
            _unsupported("LearnedSoftAggregate with a separate score basis / group_dim != 1")
        y = ops.soft_aggregate(x, self.feat2score.weight, self.feat2score.bias)
        return y.unsqueeze(1) if self.keepdim else y


class ExpandedFeatTrans(nn.Module):
    """Value projection into M modes, P.V, then (FFN) shared mid Linear + GELU, per-mode output Linear, LayerNorm
    and learned soft aggregation over the modes (reference :329-476)."""

    def __init__(self, config, name):
        super().__init__()
        self.config, self.name = config, name
        self.in_feat_dim, self.feat_dim, self.num_modes = config.in_feat_dim, config.feat_dim, config.num_modes
        self.feat_dim_allmode = self.feat_dim * self.num_modes
        self.has_FFN = config.has_FFN and not config.eval_robustness
        self.has_input_skip = getattr(config, 'has_input_skip', False)
        if self.has_input_skip:
            _unsupported("has_input_skip")
        if config.use_mince_transformer and config.mince_scales is not None:
            # (:344-354) P.V per scale on the channel windows of --minceprops, upsampled and concatenated
            _check_mince_config(config)
            self.mince_scales = list(config.mince_scales)
            self.num_scales = len(self.mince_scales)
            self.mince_channel_props = config.mince_channel_props
            self.mince_channel_indices, _ = fracs_to_indices(self.feat_dim, self.mince_channel_props)
        else:
            self.num_scales = 0
            self.mince_scales = None
        self.first_linear = nn.Linear(self.in_feat_dim, self.feat_dim_allmode, bias=config.v_has_bias)
        self.first_norm_layer = nn.LayerNorm(self.feat_dim, eps=1e-12, elementwise_affine=True)
        self.base_initializer_range = config.base_initializer_range
        self.pool_modes_keepdim = False
        self.pool_modes_feat = config.pool_modes_feat
        if self.pool_modes_feat != 'softmax':
            _unsupported("pool_modes_feat=%r" % self.pool_modes_feat)
        self.feat_softaggr = LearnedSoftAggregate(self.feat_dim, group_dim=1, keepdim=False)
        self.mid_type = config.mid_type
        if self.mid_type == 'shared':
            self.intermediate = MMSharedMid(config)
        elif self.mid_type == 'private':
            self.intermediate = MMPrivateMid(config)
        else:
            _unsupported("mid_type=%r" % self.mid_type)
        if config.trans_output_type == 'shared':
            self.output = MMSharedOutput(config)
        elif config.trans_output_type == 'private':
            self.output = MMPrivateOutput(config)

    def add_identity_bias(self):
        """W[:F,:F] <- 0.5 W[:F,:F] + 0.2 I on the value projection (reference :392-402)."""
        s = self.config.feattrans_lin1_idbias_scale
        if s > 0:
            Fd = self.feat_dim
            eye = torch.eye(Fd) * self.base_initializer_range * s
            w = self.first_linear.weight.data
            w[:Fd, :Fd] = w[:Fd, :Fd] * 0.5 + eye.to(w)

    def _can_fold(self):
        return self.has_FFN and isinstance(self.output, MMPrivateOutput) and isinstance(self.intermediate, MMSharedMid) \
            and self.first_linear.bias is None and self.first_linear.weight.shape[1] % 4 == 0 and self.feat_dim % 4 == 0

    def supports_fused_attention(self):
        """The expansion block whose P.V / mid / output chain is one autograd node (ops.attn_pv_gelu_group_linear), which
        CrossAttFeatTrans feeds with the fused attention probabilities (ops.attn_probs)."""
        return self.has_FFN and isinstance(self.output, MMPrivateOutput) and isinstance(self.intermediate, MMSharedMid)

    def _value_bank(self, input_feat, tag="big"):
        """V' = (x Wv^T) Wm^T, the value bank already pushed through MMSharedMid's Linear (see forward).  tag: precision
        class of the bank's projections (ops.small_tag of bank rows vs. query rows)."""
        M, mid = self.num_modes, self.intermediate
        B, U2 = input_feat.shape[0], input_feat.shape[1]
        if self._can_fold():
            return ops.folded_value_bank(input_feat, self.first_linear.weight, mid.shared_linear.weight, M, tag)
        v = ops.linear(input_feat, self.first_linear.weight, self.first_linear.bias, tag=tag)     # [B,U2,M*F]
        return ops.linear(v.view(B, U2, M, self.feat_dim), mid.shared_linear.weight, tag=tag).view(B, U2, M * self.feat_dim)

    def _norm_aggregate(self, y):
        p = self.output.dropout.p if self.training else 0.0
        ln = self.output.resout_norm_layer
        f2s = self.feat_softaggr.feat2score
        return ops.ln_softaggr(y, ln.weight, ln.bias, f2s.weight, f2s.bias, drop_p=p,
                               seed=ops.new_dropout_seed(y.device) if p > 0 else 0)

    def _mince_fuse(self, input_feat, probs, grid):
        """(:413-443) U [B,M,N,F]: V = first_linear(x) in full; per scale s its channel window [Lv_s, Rv_s) of every mode
        is downsampled onto the scale's grid (zero-padded to a multiple of 4 columns), multiplied by P_s and upsampled
        back into its window of U."""
        M, Fd = self.num_modes, self.feat_dim
        grids = mince_grids(grid, self.mince_scales)
        if len(probs) != self.num_scales:
            raise ValueError("ExpandedFeatTrans: %d attention probabilities for %d mince scales" % (len(probs), self.num_scales))
        idx = self.mince_channel_indices
        wins = [(idx[s], idx[s + 1]) for s in range(self.num_scales)]
        if any(b <= a for a, b in wins):
            raise ValueError("ExpandedFeatTrans: an empty mince channel window %s of %d channels" % (wins, Fd))
        v = ops.linear(input_feat, self.first_linear.weight, self.first_linear.bias, round_out=False)    # [B,N,M*F]
        ratios = [(ops.down_ratio(sc),) * len(grid) for sc in self.mince_scales]
        vs = ops.resize_tokens(v, M, grid, grids, ratios, wins)                  # [B,N_s,M*pad4(w_s)] each
        us = [ops.attn_pv(p, vv, M, round_out=False) for p, vv in zip(probs, vs)]     # [B,M,N_s,pad4(w_s)]
        return ops.resize_tokens_into(us, grid, grids, wins, Fd)                 # [B,M,N,F]

    def reads_transposed_probs(self, B, U1, U2):
        """The fused P.V' node's backward reads P^T K-major (ops.pv_gelu_kmajor): forward() then takes it as probs_t."""
        return self.supports_fused_attention() and self.num_scales == 0 and \
            ops.pv_gelu_kmajor(B, self.num_modes, U1, U2, self.feat_dim)

    def forward(self, input_feat, attention_probs, in_geoshape=None, probs_t=None):
        """input_feat [B,U2,C]; attention_probs [B,M,U1,U2] -> [B,U1,F].  With mince scales: attention_probs is the list
        of per-scale probabilities and in_geoshape the token grid.  probs_t: P^T [B,M,U2,U1] from the attention kernel,
        when reads_transposed_probs() holds."""
        M = self.num_modes
        if self.num_scales > 0:
            if in_geoshape is None:
                raise ValueError("ExpandedFeatTrans: the mince transformer needs the token grid (in_geoshape)")
            u = self._mince_fuse(input_feat, attention_probs, tuple(int(g) for g in in_geoshape))
            if not self.has_FFN:
                z = u[:, 0] if M == 1 else self.feat_softaggr(u)
                return ops.layer_norm(z, self.first_norm_layer.weight, self.first_norm_layer.bias)
            # the channel windows sit between P.V and the mid Linear: the unfolded branch below
            g = self.intermediate(u)
            return self._norm_aggregate(self.output(g, u))
        folded = self.supports_fused_attention()
        if not folded:
            v = ops.linear(input_feat, self.first_linear.weight, self.first_linear.bias)     # [B,U2,M*F]
        if not self.has_FFN:
            u = ops.attn_pv(attention_probs, v, M)                                           # [B,M,U1,F]
            # (:453) soft-aggregate over the modes — the identity for one mode, whose feat2score then gets no gradient,
            # exactly as in the reference — then first_norm_layer (:456)
            z = u[:, 0] if M == 1 else self.feat_softaggr(u)
            return ops.layer_norm(z, self.first_norm_layer.weight, self.first_norm_layer.bias)
        if folded:
            # (P V) Wm^T = P (V Wm^T): push the value bank (U2 rows) through the shared mid Linear instead of the
            # fused tokens (U1 rows), and fuse MMSharedMid's bias + GELU + dropout into the P.V epilogue.  U itself
            # is only needed by the (discarded) residual of MMPrivateOutput, so it is never materialised.
            # With a bias-free value projection the two Linears on the bank fold into one weight-space product
            # W'_m = Wm Wv_m (batch-independent), so the bank is projected once.
            mid = self.intermediate
            vp = self._value_bank(input_feat, ops.small_tag(input_feat.shape[1], attention_probs.shape[2]))
            p = mid.dropout.p if self.training else 0.0
            # ... and MMPrivateOutput's grouped Linear rides in the same autograd node (its backward fuses GELU' and
            # the dropout mask into the dG GEMM epilogue)
            gl = self.output.group_linear
            y = ops.attn_pv_gelu_group_linear(attention_probs, vp, M, mid.shared_linear.bias, p,
                                              ops.new_dropout_seed(vp.device) if p > 0 else 0, gl.weight, gl.bias,
                                              probs_t)
        else:
            u = ops.attn_pv(attention_probs, v, M)
            g = self.intermediate(u)
            y = self.output(g, u)
        return self._norm_aggregate(y)


# ---------------------------------------------------------------------------------------------------
# multi-head ablation (--multihead; reference segtran_ablation.py:93-253): parameter holders with the ablation module's
# names and creation order, built on the layer's config after MultiHeadFeatTrans has set num_modes = 1
# ---------------------------------------------------------------------------------------------------
class AblationMMSharedMid(nn.Module):
    """The ablation's MMSharedMid (segtran_ablation.py:93-121): one Linear(F->F) + erf-GELU, and no dropout."""

    def __init__(self, config):
        super().__init__()
        self.num_modes, self.feat_dim = config.num_modes, config.feat_dim
        self.shared_linear = nn.Linear(self.feat_dim, self.feat_dim)
        self.mid_act_fn = config.act_fun


class AblationMMPrivateOutput(nn.Module):
    """The ablation's MMPrivateOutput (segtran_ablation.py:125-145) with one mode: Conv1d(F, F, 1) + dropout + LayerNorm;
    the residual is computed and discarded, as in MMPrivateOutput."""

    def __init__(self, config):
        super().__init__()
        self.num_modes, self.feat_dim = config.num_modes, config.feat_dim
        fam = self.feat_dim * self.num_modes
        self.group_linear = nn.Conv1d(fam, fam, 1, groups=self.num_modes)
        self.resout_norm_layer = nn.LayerNorm(self.feat_dim, eps=1e-12, elementwise_affine=True)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class AblationMMSharedOutput(nn.Module):
    """The ablation's MMSharedOutput (segtran_ablation.py:149-178): Linear(F->F) + residual + dropout + LayerNorm; the
    residual is kept."""

    def __init__(self, config):
        super().__init__()
        self.num_modes, self.feat_dim = config.num_modes, config.feat_dim
        self.shared_linear = nn.Linear(self.feat_dim, self.feat_dim)
        self.resout_norm_layer = nn.LayerNorm(self.feat_dim, eps=1e-12, elementwise_affine=True)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class MultiHeadFeatTrans(nn.Module):
    """Multi-head attention output in place of the multi-mode expansion (reference segtran_ablation.py:183-253): the M
    attention modes are M heads of dh = F / M channels.
        V = x Wv^T + bv  [B,U2,F];  U[:, :, h*dh:(h+1)*dh] = P_h V[:, :, h*dh:(h+1)*dh];  G = gelu(U Wm^T + bm)
        'private': Y = LN(dropout(G Wo^T + bo))        'shared': Y = LN(dropout(G Ws^T + bs + U))
    -> [B,U1,F], no soft aggregation.  Not an ExpandedFeatTrans: SegtranInitWeights gives first_linear no identity bias,
    as in the reference.  Like the reference, it sets num_modes = 1 on the layer's config (its CrossAttFeatTrans has
    already read M)."""

    def __init__(self, config, name):
        super().__init__()
        self.config, self.name = config, name
        self.in_feat_dim, self.feat_dim, self.num_modes = config.in_feat_dim, config.feat_dim, config.num_modes
        if self.feat_dim % self.num_modes:
            # the reference fails at its reshape (segtran_ablation.py:239)
            raise ValueError("MultiHeadFeatTrans: feat_dim %d is not divisible by %d heads" % (self.feat_dim, self.num_modes))
        if config.mid_type != 'shared':
            _unsupported("mid_type=%r with ablate_multihead" % (config.mid_type,))
        if config.trans_output_type not in ('private', 'shared'):
            _unsupported("trans_output_type=%r" % (config.trans_output_type,))
        self.feat_dim_onehead = self.feat_dim // self.num_modes
        self.feat_dim_allhead = self.feat_dim_onehead * self.num_modes
        self.first_linear = nn.Linear(self.in_feat_dim, self.feat_dim_allhead)
        config.num_modes = 1                    # (:203) intermediate and output see one mode
        self.mid_type = config.mid_type
        self.intermediate = AblationMMSharedMid(config)
        if config.trans_output_type == 'shared':
            self.output = AblationMMSharedOutput(config)
        else:
            self.output = AblationMMPrivateOutput(config)

    def supports_fused_attention(self):
        return True

    def forward(self, input_feat, attention_probs):
        """input_feat [B,U2,C]; attention_probs [B,M,U1,U2] -> [B,U1,F] (:228-253)."""
        v = ops.linear(input_feat, self.first_linear.weight, self.first_linear.bias, tag="proj")       # [B,U2,F]
        u = ops.attn_pv(attention_probs, v, self.num_modes, heads=True)                                # [B,U1,F]
        mid = self.intermediate.shared_linear
        g = ops.linear(u, mid.weight, mid.bias, gelu=True, tag="proj")
        out = self.output
        p = out.dropout.p if self.training else 0.0
        seed = ops.new_dropout_seed(u.device) if p > 0 else 0
        if isinstance(out, AblationMMSharedOutput):
            z = ops.linear(g, out.shared_linear.weight, out.shared_linear.bias, drop_p=p, seed=seed, tag="proj",
                           round_out=False, addend=u)
        else:
            z = ops.linear(g, out.group_linear.weight, out.group_linear.bias, drop_p=p, seed=seed, tag="proj",
                           round_out=False)
        ln = out.resout_norm_layer
        return ops.layer_norm(z, ln.weight, ln.bias, round_out=False)


def _new_diag(device):
    """A layer's attention diagnostics, kept on the device: running max of the scores, clamped calls, rows where the
    reference's lower clamp could have mattered."""
    return torch.tensor([-3.0e38, 0.0, 0.0], device=device)


def _attention_probs(q, k, M, clip, drop_p, diag, *, fused, posbias=None, alpha=None, row_bias=None, tag="big",
                     kmajor_dq=False, transposed=False, key_t=None):
    """P = dropout(softmax(clamp_if(alpha Q K^T [+ row_bias]) [+ posbias])) per mode -> (P, S, amax, Pt).
    fused: one sx_attn_probs_fwd kernel (ops.attn_probs), S = amax = None; with kmajor_dq its backward's dQ = dS K reads
    a K-major copy of the keys; with transposed (and autograd recording) the kernel also writes Pt = P^T [B,M,U2,U1].
    Otherwise the raw scores S (ops.attn_scores, their maximum tracked on the device in amax; key_t: the keys'
    ops.tokens_t() twin for its dQ), then ops.softmax, and Pt = None."""
    seed = ops.new_dropout_seed(q.device) if drop_p > 0 else 0
    if fused:
        if transposed and torch.is_grad_enabled():
            P, Pt = ops.attn_probs(q, k, M, alpha, clip, drop_p, seed, diag, posbias, kmajor_dq=kmajor_dq, transposed=True)
            return P, None, None, Pt
        return ops.attn_probs(q, k, M, alpha, clip, drop_p, seed, diag, posbias, kmajor_dq=kmajor_dq), None, None, None
    amax = torch.full((1,), -3.0e38, device=q.device)
    S = ops.attn_scores(q, k, M, amax, row_bias, tag, alpha, kt=key_t)
    return ops.softmax(S, amax, clip, drop_p, seed, diag, posbias), S, amax, None


class CrossAttFeatTrans(nn.Module):
    """Cross attention with tied Q/K projection + ExpandedFeatTrans, or MultiHeadFeatTrans with ablate_multihead
    (reference :478-610)."""

    def __init__(self, config, name):
        super().__init__()
        self.config, self.name = config, name
        self.num_modes, self.in_feat_dim, self.feat_dim = config.num_modes, config.in_feat_dim, config.feat_dim
        self.attention_mode_dim = self.in_feat_dim // self.num_modes
        self.att_size_allmode = self.num_modes * self.attention_mode_dim
        self.query = nn.Linear(self.in_feat_dim, self.att_size_allmode, bias=config.qk_have_bias)
        self.key = nn.Linear(self.in_feat_dim, self.att_size_allmode, bias=config.qk_have_bias)
        self.base_initializer_range = config.base_initializer_range
        if config.pos_code_type == 'bias':
            if config.use_attn_consist_loss:
                raise NotImplementedError("segtran_b200: --attnconsist with --pos bias is not implemented (the attention "
                                          "scores this build keeps do not include the positional biases)")
            self.pos_code_weight = config.pos_code_weight
        else:
            self.pos_code_weight = 1
        if config.ablate_multihead:
            self.out_trans = MultiHeadFeatTrans(config, name)
        else:
            self.out_trans = ExpandedFeatTrans(config, name)
        self.att_dropout = nn.Dropout(config.attention_probs_dropout_prob)
        self.keep_attn_scores = config.use_attn_consist_loss
        self.tie_qk_scheme = config.tie_qk_scheme
        self.attn_clip = config.attn_clip
        self.attn_diag_cycles = config.__dict__.get('attn_diag_cycles', 500)
        self.call_count = 0
        self.attention_scores = None
        self._diag = None            # device [2]: running max of the scores, number of clamped calls

    def tie_qk(self, tie_qk_scheme=None):
        if tie_qk_scheme is not None:
            self.tie_qk_scheme = tie_qk_scheme
        if self.tie_qk_scheme == 'shared':
            self.key.weight = self.query.weight
            if self.key.bias is not None:
                self.key.bias = self.query.bias
        elif self.tie_qk_scheme == 'loose':
            self.key.weight.data.copy_(self.query.weight)
            if self.key.bias is not None:
                self.key.bias.data.copy_(self.query.bias)

    def add_identity_bias(self):
        """First d rows: W <- 0.5 W + 0.2 [I_d | I_d | ...] (reference :538-546)."""
        d = self.attention_mode_dim
        eye = torch.eye(d) * self.base_initializer_range * self.config.query_idbias_scale
        eye = eye.repeat(1, self.in_feat_dim // d)
        w = self.key.weight.data
        w[:d] = w[:d] * 0.5 + eye.to(w)

    # ---- lazily synchronised diagnostics (the reference does two .item() syncs per call, :569-573) ----
    def _diag_values(self):
        if self._diag is None:
            return 0.0, 0
        m, c = self._diag.tolist()[:2]
        return (m if m > -1e38 else 0.0), int(c)

    @property
    def lower_clamp_ambiguous_rows(self):
        """Rows of fused-attention calls where the reference's LOWER clamp could have changed the result (a row whose
        maximum is below -(clip-104) in a call whose global maximum exceeded +clip; see csrc/sx_attn.cu).  Expected 0."""
        return 0 if self._diag is None else int(self._diag.tolist()[2])

    @property
    def max_attn(self):
        return max(self._diag_values()[0], 0)

    @property
    def clamp_count(self):
        return self._diag_values()[1]

    def forward(self, in_query, in_key=None, pos_biases=None, query_t=None):
        """pos_biases: an ops.PosBias over the tokens of a self-attention (the reference's [1,1,N,N] bias matrix, kept
        as its window table); it is added to the scores after the clamp, scaled by pos_code_weight (:589-592).
        query_t: in_query's ops.tokens_t() twin (or None), for the query projection's weight gradient."""
        if in_key is None:
            in_key = in_query
        pb = None
        if pos_biases is not None:
            if not isinstance(pos_biases, ops.PosBias):
                raise TypeError("CrossAttFeatTrans: pos_biases must be an ops.PosBias (SlidingPosBiases2D/3D output)")
            if self.keep_attn_scores:
                raise NotImplementedError("segtran_b200: --attnconsist with --pos bias is not implemented")
            if in_query.shape[1] != pos_biases.num_tokens or in_key.shape[1] != pos_biases.num_tokens:
                raise ValueError("CrossAttFeatTrans: positional biases over %s cells need a self-attention over as many "
                                 "tokens (got %d queries, %d keys)" % (pos_biases.grid, in_query.shape[1], in_key.shape[1]))
            pb = pos_biases.with_weight(float(self.pos_code_weight))
        M = self.num_modes
        # precision classes (ops.small_tag): the projection of the shorter side is an attractor-row product when that side is
        # at most a quarter of the other one; everything else is a token-row projection
        nq, nk = in_query.shape[1], in_key.shape[1]
        tq = ops.small_tag(nq, nk) if nq < nk else "proj"
        tk = ops.small_tag(nk, nq) if nk < nq else "proj"
        q = ops.linear(in_query, self.query.weight, self.query.bias, tag=tq, xt=query_t)
        k = ops.linear(in_key, self.key.weight, self.key.bias, tag=tk)
        dev = q.device
        if self._diag is None or self._diag.device != dev:
            self._diag = _new_diag(dev)
        p = self.att_dropout.p if self.training else 0.0
        diag_call = self.training and (self.call_count + 1) % self.attn_diag_cycles == 0     # prints avg-attn: needs S
        fused = ops.attn_fusion_enabled() and not self.keep_attn_scores and not diag_call and q.is_cuda and \
            self.attention_mode_dim % 4 == 0 and self.out_trans.supports_fused_attention()
        # the expansion block's dQ = dS K reads a K-major copy of the keys (the squeeze-out's attractor keys are small
        # against dS); multi-head reads its keys in place (DESIGN §4.3).  When the expansion block's dV' = P^T dH reads
        # K-major operands, the attention kernel also writes P^T for it.
        expanded = isinstance(self.out_trans, ExpandedFeatTrans)
        transposed = fused and expanded and self.out_trans.reads_transposed_probs(k.shape[0], nq, nk)
        probs, s, amax, probs_t = _attention_probs(q, k, M, float(self.attn_clip), p, self._diag, fused=fused,
                                                   posbias=pb, kmajor_dq=expanded, transposed=transposed)
        # kept after the conditional clamp, as the reference keeps them (:578-598)
        self.attention_scores = ops.clamp_if(s, amax, float(self.attn_clip)) if self.keep_attn_scores else None
        if self.training:
            self.call_count += 1
            if self.call_count % self.attn_diag_cycles == 0:        # never on the fused path: diag_call above
                with torch.no_grad():
                    avg = float(s.sum() / (s > 0).sum().clamp_min(1))
                mx, cc = self._diag_values()
                print("max-attn: {:.2f}, avg-attn: {:.2f}, clamp-count: {}".format(mx, avg, cc))
                self._diag = _new_diag(dev)
        if probs_t is not None:
            return self.out_trans(in_key, probs, probs_t=probs_t)
        return self.out_trans(in_key, probs)


class CrossMinceAttFeatTrans(nn.Module):
    """Mince attention (reference :612-785): per scale s, the Q/K channel window [L_s, R_s) of every mode (the modes'
    d = in_feat_dim / M channels split equally between the scales) is downsampled onto the scale's grid (scale_factor
    1/scale_s), S_s = Q_s K_s^T / sqrt(d) with the FULL d, conditionally clamped on this scale's own maximum, plus
    pos_code_weight * the scale's positional biases, softmax and attention dropout; then ExpandedFeatTrans combines the
    scales (:404-447).  Not a CrossAttFeatTrans: SegtranInitWeights leaves query and key untied and gives the key no
    identity bias."""

    def __init__(self, config, name):
        super().__init__()
        self.config, self.name = config, name
        self.num_modes, self.in_feat_dim, self.feat_dim = config.num_modes, config.in_feat_dim, config.feat_dim
        self.attention_mode_dim = self.in_feat_dim // self.num_modes
        self.att_size_allmode = self.num_modes * self.attention_mode_dim
        self.query = nn.Linear(self.in_feat_dim, self.att_size_allmode, bias=config.qk_have_bias)
        self.key = nn.Linear(self.in_feat_dim, self.att_size_allmode, bias=config.qk_have_bias)
        if not config.use_mince_transformer:
            raise ValueError("CrossMinceAttFeatTrans needs use_mince_transformer")
        _check_mince_config(config)
        self.mince_scales = list(config.mince_scales)
        self.num_scales = len(self.mince_scales)
        self.mince_qk_channel_indices, _ = fracs_to_indices(self.attention_mode_dim, [1] * self.num_scales)
        if any(self.mince_qk_channel_indices[s + 1] <= self.mince_qk_channel_indices[s] for s in range(self.num_scales)):
            raise ValueError("CrossMinceAttFeatTrans: %d channels per mode cannot be split between %d scales"
                             % (self.attention_mode_dim, self.num_scales))
        self.base_initializer_range = config.base_initializer_range
        self.pos_code_weight = config.pos_code_weight if config.pos_code_type == 'bias' else 1
        if config.ablate_multihead:
            _unsupported("ablate_multihead")
        if config.use_attn_consist_loss:
            raise NotImplementedError("segtran_b200: --attnconsist with --mince is not implemented (the reference "
                                      "crashes on the per-scale list of attention scores)")
        self.out_trans = ExpandedFeatTrans(config, name)
        self.att_dropout = nn.Dropout(config.attention_probs_dropout_prob)
        self.keep_attn_scores = False
        self.tie_qk_scheme = config.tie_qk_scheme
        self.attn_clip = config.attn_clip
        self.attn_diag_cycles = config.__dict__.get('attn_diag_cycles', 500)
        self.call_count = 0
        self.attention_scores = None
        self._diag = None            # per scale, device [3]: running max of the scores, clamped calls, ambiguous rows

    tie_qk = CrossAttFeatTrans.tie_qk
    add_identity_bias = CrossAttFeatTrans.add_identity_bias

    # ---- per-scale diagnostics, synchronised lazily (the reference does .item() syncs per scale, :738-755) ----
    def _diag_lists(self):
        if self._diag is None:
            return [0.0] * self.num_scales, [0] * self.num_scales, [0] * self.num_scales
        vals = [d.tolist() for d in self._diag]
        return [max(v[0], 0.0) for v in vals], [int(v[1]) for v in vals], [int(v[2]) for v in vals]

    @property
    def max_attn(self):
        return self._diag_lists()[0]

    @property
    def clamp_count(self):
        return self._diag_lists()[1]

    @property
    def lower_clamp_ambiguous_rows(self):
        """Rows where the reference's lower clamp could have changed the result, summed over the scales (expected 0)."""
        return sum(self._diag_lists()[2])

    def forward(self, in_query, query_geoshape, in_key=None, key_geoshape=None, pos_biases=None):
        """in_query [B,N,C] on the token grid query_geoshape; pos_biases: None or one ops.PosBias (or None) per scale, each
        over that scale's grid."""
        if in_key is None:
            in_key, key_geoshape = in_query, query_geoshape
        grid = tuple(int(g) for g in query_geoshape)
        if key_geoshape is None or tuple(int(g) for g in key_geoshape) != grid:
            raise ValueError("CrossMinceAttFeatTrans: query and key grids must agree (got %s and %s)"
                             % (grid, None if key_geoshape is None else tuple(key_geoshape)))
        grids = mince_grids(grid, self.mince_scales)
        N = _prod(grid)
        if in_query.shape[1] != N or in_key.shape[1] != N:
            raise ValueError("CrossMinceAttFeatTrans: %d / %d tokens on a grid of %d cells"
                             % (in_query.shape[1], in_key.shape[1], N))
        pbs = [None] * self.num_scales
        if pos_biases is not None:
            if len(pos_biases) != self.num_scales:
                raise ValueError("CrossMinceAttFeatTrans: %d positional biases for %d scales"
                                 % (len(pos_biases), self.num_scales))
            for s, pb in enumerate(pos_biases):
                if pb is None:
                    continue
                if not isinstance(pb, ops.PosBias):
                    raise TypeError("CrossMinceAttFeatTrans: pos_biases entries must be ops.PosBias or None")
                if pb.grid != grids[s]:
                    raise ValueError("CrossMinceAttFeatTrans: positional biases over %s at scale %s, whose grid is %s"
                                     % (pb.grid, self.mince_scales[s], grids[s]))
                pbs[s] = pb.with_weight(float(self.pos_code_weight))
        M, d = self.num_modes, self.attention_mode_dim
        q = ops.linear(in_query, self.query.weight, self.query.bias, tag="proj", round_out=False)
        k = ops.linear(in_key, self.key.weight, self.key.bias, tag="proj", round_out=False)
        idx = self.mince_qk_channel_indices
        wins = [(idx[s], idx[s + 1]) for s in range(self.num_scales)]
        ratios = [(ops.down_ratio(sc),) * len(grid) for sc in self.mince_scales]
        qs = ops.resize_tokens(q, M, grid, grids, ratios, wins)        # [B,N_s,M*pad4(w_s)], TF32-rounded
        ks = ops.resize_tokens(k, M, grid, grids, ratios, wins)
        dev = q.device
        if self._diag is None or self._diag[0].device != dev:
            self._diag = [_new_diag(dev) for _ in range(self.num_scales)]
        p = self.att_dropout.p if self.training else 0.0
        alpha = 1.0 / math.sqrt(d)                                     # (:736) the full per-mode width
        self.call_count += 1
        diag_call = self.training and self.call_count % self.attn_diag_cycles == 0     # prints avg-attn: needs S
        fused = ops.attn_fusion_enabled() and not diag_call and q.is_cuda
        probs = []
        for s in range(self.num_scales):
            P, sc, _, _ = _attention_probs(qs[s], ks[s], M, float(self.attn_clip), p, self._diag[s], fused=fused,
                                        posbias=pbs[s], alpha=alpha)  # [B,M,N_s,N_s]
            probs.append(P)
            if diag_call:
                with torch.no_grad():
                    avg = float(sc.sum() / (sc > 0).sum().clamp_min(1))
                mx, cc, _ = self._diag_lists()
                print("{} attn max: {:.2f}, avg: {:.2f}, clamp-count: {}".format(self.mince_scales[s], mx[s], avg, cc[s]))
                self._diag[s] = _new_diag(dev)
        return self.out_trans(in_key, probs, grid)


class SqueezedAttFeatTrans(nn.Module):
    """Squeezed attention: A learned attractors attend to the N tokens (1 mode, no FFN), then the tokens attend to
    the updated attractors (M modes, full expansion block) — O(N*A) (reference :787-816)."""

    def __init__(self, config, name):
        super().__init__()
        self.config, self.name = config, name
        self.in_feat_dim, self.num_attractors = config.in_feat_dim, config.num_attractors
        if config.use_mince_transformer:
            _unsupported("the mince transformer")
        if config.ablate_multihead:
            raise NotImplementedError("segtran_b200: ablate_multihead with squeezed attention is not implemented (the "
                                      "reference crashes there: MultiHeadFeatTrans reshapes the attractor-side output "
                                      "with the token count, segtran_ablation.py:239; its drivers turn --multihead into "
                                      "--nosqueeze)")
        config1 = copy.copy(config)
        config1.feat_dim = config1.in_feat_dim
        config1.num_modes = 1
        config1.has_FFN = config.has_FFN_in_squeeze
        self.in_ator_trans = CrossAttFeatTrans(config1, name + '-in-squeeze')
        self.ator_out_trans = CrossAttFeatTrans(config, name + '-squeeze-out')
        self.attractors = nn.Parameter(torch.randn(1, self.num_attractors, self.in_feat_dim))
        self.attention_scores = None

    def _in_squeeze_reassociated(self, in_feat, ht):
        """In-squeeze (reference :813 -> CrossAttFeatTrans.forward with M=1, no FFN) with the two token-sized
        projections re-associated away (SURVEY §7): with Q1 = Att Wq^T + bq,
            S1 = Q1 (h Wk^T + bk)^T / sqrt(C) = ((Q1 Wk) h^T + (Q1 . bk) 1^T) / sqrt(C)
            Z  = P1 (h Wv^T)                  = (P1 h) Wv^T
        so the [N x C x C] key and value GEMMs become [A x C x C] ones; exact up to fp rounding.
        ht: in_feat's ops.tokens_t() twin (or None), read K-major by P1 h and by the backward's dS1 h."""
        t = self.in_ator_trans
        C = self.in_feat_dim
        st = ops.small_tag(self.num_attractors, in_feat.shape[1])
        x3 = ops.rt_for(st) == 0              # the attractor-row chain runs as 3-pass products: keep q1 unrounded for it
        q1 = ops.linear(self.attractors, t.query.weight, t.query.bias, tag=st, round_out=not x3)   # [1,A,C]
        qw = ops.linear(q1, t.key.weight.t(), tag=st)                                 # Q1 Wk            [1,A,C]
        rb = None
        if t.key.bias is not None:                                                    # (Q1 . bk) / sqrt(C)  [A]
            rb = ops.scale(ops.matvec(q1[0], t.key.bias), 1.0 / math.sqrt(C))
        dev = in_feat.device
        if t._diag is None or t._diag.device != dev:
            t._diag = _new_diag(dev)
        p = t.att_dropout.p if t.training else 0.0
        probs, s, amax, _ = _attention_probs(qw, in_feat, 1, float(t.attn_clip), p, t._diag, fused=False, row_bias=rb,
                                             tag="insq", key_t=ht)                     # [B,1,A,N]
        t.attention_scores = ops.clamp_if(s, amax, float(t.attn_clip)) if t.keep_attn_scores else None
        if t.training:
            t.call_count += 1
        u = ops.attn_pv(probs, in_feat, 1, tag="insq", round_out=not x3, vt=ht)        # P1 h            [B,1,A,C]
        ot = t.out_trans
        z = ops.linear(u[:, 0], ot.first_linear.weight, tag=st, round_out=False)       # (P1 h) Wv^T     [B,A,C]
        # the updated attractors feed the squeeze-out key projection and the value bank (same precision class)
        return ops.layer_norm(z, ot.first_norm_layer.weight, ot.first_norm_layer.bias, consumer_tag=st)

    def forward(self, in_feat, pos_biases=None):
        if pos_biases is not None:
            _unsupported("positional biases with squeezed attention")
        t = self.in_ator_trans
        ht = None
        if t.num_modes == 1 and not t.out_trans.has_FFN and t.out_trans.first_linear.bias is None \
                and t.feat_dim == self.in_feat_dim:
            # the tokens transposed once, when the in-squeeze's token contractions read them K-major: P1 h and dS1 h
            # per sample, and the squeeze-out query projection's weight gradient over all B*N token rows
            ht = ops.tokens_t(in_feat, self.num_attractors, "insq")
            att = self._in_squeeze_reassociated(in_feat, ht)
        else:
            att = t(self.attractors, in_feat)       # attractors are batch-invariant: projected once
        ops.grad_ready(att, self.ator_out_trans.parameters())       # backward past `att`: the squeeze-out weights are final
        out = self.ator_out_trans(in_feat, att, query_t=ht)
        self.attention_scores = self.ator_out_trans.attention_scores
        return out


class LearnedSinuPosEmbedder(nn.Module):
    """Learnable sinusoid code: Linear(pd->C), sin/cos interleaved, LayerNorm (reference :979-998)."""

    def __init__(self, pos_dim, pos_embed_dim, omega=1, affine=False):
        super().__init__()
        self.pos_dim, self.pos_embed_dim, self.omega = pos_dim, pos_embed_dim, omega
        if omega != 1 or affine:
            _unsupported("LearnedSinuPosEmbedder with omega != 1 or affine")
        self.pos_fc = nn.Linear(pos_dim, pos_embed_dim, bias=True)
        self.pos_mix_norm_layer = nn.LayerNorm(pos_embed_dim, eps=1e-12, elementwise_affine=affine)

    def forward(self, pos_normed):
        """pos_normed [..., pd] (already divided by its maximum, as SegtranPosEncoder does) -> [..., C] (reference :989-998)."""
        shp = pos_normed.shape
        pe = ops.pos_code(pos_normed.reshape(-1, shp[-1]), self.pos_fc.weight, self.pos_fc.bias, normalize=False)
        return pe.view(*shp[:-1], -1)


class NoneEmbedder(nn.Module):
    """pos_code_type 'none': no positional code at all (reference segtran_ablation.py:68-74)."""

    def forward(self, pos_normed):
        return None


class _SlidingPosBiases(nn.Module):
    """Sliding-window positional biases (reference SlidingPosBiases2D/3D, segtran_shared.py:1002-1175): one learned
    `biases` table [2R+1]^pd, zero-initialised.  The query at cell q and the key at cell k (row-major cells of the
    feature grid) get biases[k - q + R] when |k_i - q_i| <= R in every dimension, else 0.
    The reference expands the table into an [N,N] matrix through persistent int64 index buffers (all_h1s, ...: 1.3 GB
    at the 3-D default max_pos_size); here forward returns the table and the grid (ops.PosBias), and the attention
    kernels read the table directly.  Those buffers are not allocated: a reference checkpoint's all_* entries are
    accepted and dropped on load, and this module's state_dict is the reference's minus them."""

    _INDEX_BUFFERS = ()

    def __init__(self, pos_dim, pos_bias_radius, max_pos_size):
        super().__init__()
        if pos_dim != self._POS_DIM:
            raise ValueError("%s: pos_dim must be %d" % (type(self).__name__, self._POS_DIM))
        if pos_bias_radius < 1:
            raise ValueError("%s: pos_bias_radius must be >= 1 (got %d)" % (type(self).__name__, pos_bias_radius))
        self.pos_dim = pos_dim
        self.R = pos_bias_radius
        self.max_pos_size = tuple(int(m) for m in max_pos_size)
        self.biases = nn.Parameter(torch.zeros([2 * pos_bias_radius + 1] * pos_dim))

    def forward(self, feat_shape, device=None, table=None):
        """feat_shape: the token grid (its last pos_dim extents) -> ops.PosBias with weight 1 (CrossAttFeatTrans applies
        pos_code_weight).  table: a stand-in for `biases` (the eval-mode snapshot of SegtranPosEncoder)."""
        grid = tuple(int(s) for s in tuple(feat_shape)[-self.pos_dim:])
        if any(g > m for g, m in zip(grid, self.max_pos_size)):
            raise ValueError("%s: feature grid %s exceeds max_pos_size %s" % (type(self).__name__, grid, self.max_pos_size))
        return ops.PosBias(self.biases if table is None else table, self.R, grid, 1.0)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        for name in self._INDEX_BUFFERS:
            state_dict.pop(prefix + name, None)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)


class SlidingPosBiases2D(_SlidingPosBiases):
    _POS_DIM = 2
    _INDEX_BUFFERS = ('all_h1s', 'all_w1s', 'all_h2s', 'all_w2s')

    def __init__(self, pos_dim, pos_bias_radius=7, max_pos_size=(100, 100)):
        super().__init__(pos_dim, pos_bias_radius, max_pos_size)


class SlidingPosBiases3D(_SlidingPosBiases):
    _POS_DIM = 3
    _INDEX_BUFFERS = ('all_h1s', 'all_w1s', 'all_d1s', 'all_h2s', 'all_w2s', 'all_d2s')

    def __init__(self, pos_dim, pos_bias_radius=7, max_pos_size=(20, 20, 20)):
        super().__init__(pos_dim, pos_bias_radius, max_pos_size)


class SegtranPosEncoder(nn.Module):
    """pos / pos.max() -> learnable sinusoid code ('lsinu'), sliding-window biases ('bias') or nothing ('none'); cached
    in eval mode (reference :1177-1238)."""

    def __init__(self, config):
        super().__init__()
        self.feat_dim = config.trans_in_dim
        self.pos_embed_dim = self.feat_dim
        self.pos_code_type = config.pos_code_type
        if self.pos_code_type == 'lsinu':
            self.pos_coder = LearnedSinuPosEmbedder(config.pos_dim, self.pos_embed_dim, omega=1, affine=False)
        elif self.pos_code_type == 'none':
            self.pos_coder = NoneEmbedder()
        elif self.pos_code_type == 'bias':
            cls = {2: SlidingPosBiases2D, 3: SlidingPosBiases3D}.get(config.pos_dim)
            if cls is None:
                raise ValueError("SegtranPosEncoder: positional biases need pos_dim 2 or 3 (got %r)" % config.pos_dim)
            self.pos_coder = cls(config.pos_dim, config.pos_bias_radius, config.max_pos_size)
        else:
            _unsupported("pos_code_type=%r" % self.pos_code_type)
        self.cached_pos_code = None
        self.cached_feat_shape = None

    def forward(self, orig_feat_shape, voxels_pos):
        """'lsinu': voxels_pos [B,N,pd] -> code [N,C0] when the batch shares one set of positions (stride-0 batch dim or
        B == 1), else [B,N,C0].  The global max of the whole tensor normalises the positions (:1231).
        'bias': -> ops.PosBias over the grid orig_feat_shape.  A forward that can differentiate (training, or eval with
        grad enabled) reads the live table, so `biases` gets its gradient, and caches a snapshot of the values it read.
        An eval pass under no_grad on the same feature shape reuses that snapshot; a new shape snapshots the table afresh
        (:1209-1215).  So inference right after training sees the table of the last training forward, as the reference's
        cached [N,N] matrix does; like the lsinu cache, a code that would carry a graph is rebuilt rather than
        re-used.  'none': -> None."""
        if self.pos_code_type == 'none':
            return None
        if self.pos_code_type == 'bias':
            key = tuple(int(s) for s in orig_feat_shape)
            if self.training or (torch.is_grad_enabled() and self.pos_coder.biases.requires_grad):
                self.cached_pos_code = self.pos_coder(key, table=self.pos_coder.biases.detach().clone())
                self.cached_feat_shape = key
                return self.pos_coder(key)
            if self.cached_pos_code is None or self.cached_feat_shape != key:
                self.cached_pos_code = self.pos_coder(key, table=self.pos_coder.biases.detach().clone())
                self.cached_feat_shape = key
            return self.cached_pos_code
        key = tuple(voxels_pos.shape)              # shape-keyed like the reference's cache (:1219)
        if not self.training and self.cached_pos_code is not None and self.cached_feat_shape == key and \
                not (torch.is_grad_enabled() and self.cached_pos_code.requires_grad):
            return self.cached_pos_code        # (a cached code that still carries a graph is rebuilt, not re-used)
        B, N, pd = voxels_pos.shape
        shared = B == 1 or voxels_pos.stride(0) == 0
        pos2d = voxels_pos[0] if shared else voxels_pos.reshape(B * N, pd)
        pe = ops.pos_code(pos2d, self.pos_coder.pos_fc.weight, self.pos_coder.pos_fc.bias)
        if not shared:
            pe = pe.view(B, N, -1)
        self.cached_pos_code, self.cached_feat_shape = pe, key
        return pe


class SegtranFusionEncoder(nn.Module):
    """The multi-layer Squeeze-and-Expansion stack (reference :819-975).  forward(vfeat [B,N,C0], voxels_pos
    [B,N,pd], vmask [B,N,1], orig_feat_shape) -> [B,N,C_last]."""

    def __init__(self, config, name):
        super().__init__()
        self.name = name
        self.num_translayers = config.num_translayers
        self.pos_code_type = config.pos_code_type
        self.translayer_compress_ratios = config.translayer_compress_ratios
        self.translayer_dims = config.translayer_dims
        self.dropout = nn.Dropout(config.hidden_dropout_prob)
        self.use_squeezed_transformer = config.use_squeezed_transformer
        self.use_mince_transformer = config.use_mince_transformer
        if self.use_squeezed_transformer and self.use_mince_transformer:
            print("Squeezed transformer cannot be used with Mince transformer.")
            print("Please specify '--nosqueeze' to disable squeezed transformer.")
            exit(0)
        if self.use_squeezed_transformer and self.pos_code_type == 'bias':
            print("Squeezed transformer cannot use Positional Biases.")
            print("Please specify '--nosqueeze' to disable squeezed transformer.")
            exit(0)
        if self.pos_code_type == 'bias' and config.use_attn_consist_loss:
            raise NotImplementedError("segtran_b200: --attnconsist with --pos bias is not implemented (the attention "
                                      "scores this build keeps do not include the positional biases)")
        # with sliding-window biases the code is not added to the features (:847-850)
        self.pos_code_weight = config.pos_code_weight if self.pos_code_type != 'bias' else 0
        if self.use_mince_transformer:
            _check_mince_config(config)
            if config.use_attn_consist_loss:
                raise NotImplementedError("segtran_b200: --attnconsist with --mince is not implemented (the reference "
                                          "crashes on the per-scale list of attention scores)")
            self.num_scales = len(config.mince_scales)
            self.mince_scales = list(config.mince_scales)
        else:
            self.num_scales = 0
        if self.num_scales > 0 and self.pos_code_type in ('bias', 'none'):
            # (:852-861) one positional encoder per scale, each over that scale's grid
            self.pos_code_layers = nn.ModuleList([SegtranPosEncoder(config) for _ in range(self.num_scales)])
        else:
            self.pos_code_layer = SegtranPosEncoder(config)
        if self.use_squeezed_transformer:
            layer_cls = SqueezedAttFeatTrans
        else:
            layer_cls = CrossMinceAttFeatTrans if self.use_mince_transformer else CrossAttFeatTrans
        layers = []
        for i in range(self.num_translayers):
            cfg_i = copy.copy(config)
            cfg_i.in_feat_dim = self.translayer_dims[i]
            cfg_i.feat_dim = self.translayer_dims[i + 1]
            layers.append(layer_cls(cfg_i, '%s%d' % (name, i)))
        self.translayers = nn.ModuleList(layers)
        self.comb_norm_layers = nn.ModuleList(
            [nn.LayerNorm(d, eps=1e-12, elementwise_affine=False) for d in self.translayer_dims[:-1]])
        self.vfeat_norm_layers = nn.ModuleList(
            [nn.LayerNorm(d, eps=1e-12, elementwise_affine=True) for d in self.translayer_dims[:-1]])
        self.use_attn_consist_loss = config.use_attn_consist_loss
        if self.use_attn_consist_loss:
            if config.use_squeezed_transformer:
                self.attn_scaler = nn.ModuleList([nn.Conv2d(1, 1, 1), nn.Conv2d(config.num_modes, 1, 1)])
            else:
                self.attn_scaler = nn.Conv2d(config.num_modes, 1, 1)
        self.layers_vfeat = []
        self.layers_attn_scores = None

    def forward(self, vfeat, voxels_pos, vmask, orig_feat_shape):
        self.layers_vfeat = []
        self.layers_attn_scores = [] if self.use_attn_consist_loss else None
        B, N, _ = vfeat.shape
        mask = vmask.reshape(B * N).to(torch.float32).contiguous() if vmask is not None else None
        x = vfeat if vfeat.dtype == torch.float32 else vfeat.float()
        if self.training and x.is_cuda:
            ops.advance_seed(x.device)           # one new dropout stream per training step (device side, graph safe)
        per_scale = self.num_scales > 0 and self.pos_code_type in ('bias', 'none')
        for i, layer in enumerate(self.translayers):
            if per_scale:
                grids = mince_grids(orig_feat_shape, self.mince_scales)
                pe = [self.pos_code_layers[s](grids[s], voxels_pos) for s in range(self.num_scales)]
            else:
                pe = self.pos_code_layer(orig_feat_shape, voxels_pos)
            ln = self.vfeat_norm_layers[i]
            p = self.dropout.p if (self.training and i == 0) else 0.0
            # 'bias' / 'none': no code on the features and no comb_norm_layers LayerNorm (:929-940); the biases (shared
            # by every layer) go into the attention scores instead
            feat_pe = pe if self.pos_code_type == 'lsinu' else None
            h = ops.prologue(x, ln.weight, ln.bias, feat_pe, float(self.pos_code_weight), mask, p,
                             ops.new_dropout_seed(x.device) if p > 0 else 0)
            ops.grad_ready(h, layer.parameters())                   # backward past `h`: this layer's weights are final
            if self.num_scales > 0:
                x = layer(h, orig_feat_shape, pos_biases=pe if self.pos_code_type == 'bias' else None)
            else:
                x = layer(h, pos_biases=pe if self.pos_code_type == 'bias' else None)
            self.layers_vfeat.append(x)
            if self.use_attn_consist_loss:
                if self.use_squeezed_transformer:
                    self.layers_attn_scores.append([self.attn_scaler[0](layer.in_ator_trans.attention_scores),
                                                    self.attn_scaler[1](layer.ator_out_trans.attention_scores)])
                else:
                    self.layers_attn_scores.append(self.attn_scaler(layer.attention_scores))
        self.orig_feat_shape = orig_feat_shape
        return x


class SegtranInitWeights(nn.Module):
    """Weight init + Q/K tying + identity bias, applied via ``self.apply`` by the shells (reference :1241-1264)."""

    def __init__(self, config, *inputs, **kwargs):
        super().__init__()
        self.config = config

    def init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            if (np.array(module.weight.shape) < self.config.min_feat_dim).all():
                print("Skip init of Linear weight %s" % (list(module.weight.shape)))
            else:
                module.weight.data.normal_(mean=0.0, std=self.config.base_initializer_range)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    def tie_qk(self, module):
        if isinstance(module, CrossAttFeatTrans) and module.tie_qk_scheme != 'none':
            module.tie_qk()

    def add_identity_bias(self, module):
        if isinstance(module, (CrossAttFeatTrans, ExpandedFeatTrans)):
            module.add_identity_bias()
