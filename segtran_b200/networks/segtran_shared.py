"""H100-native Squeeze-and-Expansion transformer stack — drop-in module surface.

Mirrors the nn.Module contract of the reference's ``code/networks/segtran_shared.py`` (class names,
constructor signatures, sub-module / parameter names and creation order, so that
``torch.manual_seed(s)`` + construction gives the reference's initial weights and reference
checkpoints load with ``load_state_dict``), while every forward runs on the sm_90a kernels in
``segtran_b200/csrc`` through ``segtran_b200.ops``.  There is no PyTorch fallback inside the stack.

Supported configuration = the one the reference's drivers force (train3d.py:174-178, train2d.py:245-249):
squeezed attention (or plain cross attention), pos_code_type 'lsinu', mid_type 'shared',
trans_output_type 'private'|'shared', tie_qk 'shared'|'loose'|'none', pool_modes_feat 'softmax', plus
--nosqueeze and --squeezeuseffn.  Ablation-only
switches (mince, sliding biases, multihead, rand/sinu/none position codes) raise NotImplementedError.
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
            _unsupported("the mince transformer")
        self.num_scales = 0
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
        """The expansion block whose P.V / mid / output chain hangs off one autograd node (ops.squeeze_out_fused)."""
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

    def forward_from_qk(self, input_feat, q, k, clip, att_p, diag):
        """Fused attention entry: q [Bq,U1,M*d], k [B,U2,M*d] (projected, TF32-rounded) instead of the probabilities —
        scores, clamp, softmax and attention dropout run inside ops.squeeze_out_fused (csrc/sx_attn.cu)."""
        mid = self.intermediate
        vp = self._value_bank(input_feat, ops.small_tag(input_feat.shape[1], q.shape[1]))
        p = mid.dropout.p if self.training else 0.0
        gl = self.output.group_linear
        dev = vp.device
        y = ops.squeeze_out_fused(q, k, vp, self.num_modes, clip, att_p, ops.new_dropout_seed(dev) if att_p > 0 else 0,
                                  mid.shared_linear.bias, p, ops.new_dropout_seed(dev) if p > 0 else 0, gl.weight, gl.bias,
                                  diag)
        return self._norm_aggregate(y)

    def forward(self, input_feat, attention_probs, in_geoshape=None):
        """input_feat [B,U2,C]; attention_probs [B,M,U1,U2] -> [B,U1,F]."""
        M = self.num_modes
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
                                              ops.new_dropout_seed(vp.device) if p > 0 else 0, gl.weight, gl.bias)
        else:
            u = ops.attn_pv(attention_probs, v, M)
            g = self.intermediate(u)
            y = self.output(g, u)
        return self._norm_aggregate(y)


class CrossAttFeatTrans(nn.Module):
    """Cross attention with tied Q/K projection + ExpandedFeatTrans (reference :478-610)."""

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
            _unsupported("pos_code_type='bias'")
        self.pos_code_weight = 1
        if config.ablate_multihead:
            _unsupported("ablate_multihead")
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

    def forward(self, in_query, in_key=None, pos_biases=None):
        if pos_biases is not None:
            _unsupported("positional biases")
        if in_key is None:
            in_key = in_query
        M = self.num_modes
        # precision classes (ops.small_tag): the projection of the shorter side is an attractor-row product when that side is
        # at most a quarter of the other one; everything else is a token-row projection
        nq, nk = in_query.shape[1], in_key.shape[1]
        tq = ops.small_tag(nq, nk) if nq < nk else "proj"
        tk = ops.small_tag(nk, nq) if nk < nq else "proj"
        q = ops.linear(in_query, self.query.weight, self.query.bias, tag=tq)
        k = ops.linear(in_key, self.key.weight, self.key.bias, tag=tk)
        dev = q.device
        if self._diag is None or self._diag.device != dev:
            self._diag = torch.tensor([-3.0e38, 0.0, 0.0], device=dev)
        p = self.att_dropout.p if self.training else 0.0
        diag_call = self.training and (self.call_count + 1) % self.attn_diag_cycles == 0     # prints avg-attn: needs S
        if ops.attn_fusion_enabled() and not self.keep_attn_scores and not diag_call and q.is_cuda and \
                self.attention_mode_dim % 4 == 0 and self.out_trans.supports_fused_attention():
            # fused squeeze-out attention: scores / clamp / softmax / dropout inside one wgmma kernel
            self.attention_scores = None
            if self.training:
                self.call_count += 1
            return self.out_trans.forward_from_qk(in_key, q, k, float(self.attn_clip), p, self._diag)
        amax = torch.full((1,), -3.0e38, device=dev)
        s = ops.attn_scores(q, k, M, amax)                                   # [B,M,U1,U2], max tracked on device
        probs = ops.softmax(s, amax, float(self.attn_clip), p, ops.new_dropout_seed(dev) if p > 0 else 0, self._diag)
        self.attention_scores = s if self.keep_attn_scores else None
        if self.training:
            self.call_count += 1
            if self.call_count % self.attn_diag_cycles == 0:
                with torch.no_grad():
                    avg = float(s.sum() / (s > 0).sum().clamp_min(1))
                mx, cc = self._diag_values()
                print("max-attn: {:.2f}, avg-attn: {:.2f}, clamp-count: {}".format(mx, avg, cc))
                self._diag = torch.tensor([-3.0e38, 0.0, 0.0], device=dev)
        return self.out_trans(in_key, probs)


class CrossMinceAttFeatTrans(nn.Module):
    def __init__(self, config, name):
        super().__init__()
        _unsupported("the mince transformer")


class SqueezedAttFeatTrans(nn.Module):
    """Squeezed attention: A learned attractors attend to the N tokens (1 mode, no FFN), then the tokens attend to
    the updated attractors (M modes, full expansion block) — O(N*A) (reference :787-816)."""

    def __init__(self, config, name):
        super().__init__()
        self.config, self.name = config, name
        self.in_feat_dim, self.num_attractors = config.in_feat_dim, config.num_attractors
        if config.use_mince_transformer:
            _unsupported("the mince transformer")
        config1 = copy.copy(config)
        config1.feat_dim = config1.in_feat_dim
        config1.num_modes = 1
        config1.has_FFN = config.has_FFN_in_squeeze
        self.in_ator_trans = CrossAttFeatTrans(config1, name + '-in-squeeze')
        self.ator_out_trans = CrossAttFeatTrans(config, name + '-squeeze-out')
        self.attractors = nn.Parameter(torch.randn(1, self.num_attractors, self.in_feat_dim))
        self.attention_scores = None

    def _in_squeeze_reassociated(self, in_feat):
        """In-squeeze (reference :813 -> CrossAttFeatTrans.forward with M=1, no FFN) with the two token-sized
        projections re-associated away (SURVEY §7): with Q1 = Att Wq^T + bq,
            S1 = Q1 (h Wk^T + bk)^T / sqrt(C) = ((Q1 Wk) h^T + (Q1 . bk) 1^T) / sqrt(C)
            Z  = P1 (h Wv^T)                  = (P1 h) Wv^T
        so the [N x C x C] key and value GEMMs become [A x C x C] ones; exact up to fp rounding."""
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
            t._diag = torch.tensor([-3.0e38, 0.0, 0.0], device=dev)
        amax = torch.full((1,), -3.0e38, device=dev)
        s = ops.attn_scores(qw, in_feat, 1, amax, rb, tag="insq")                      # [B,1,A,N]
        p = t.att_dropout.p if t.training else 0.0
        probs = ops.softmax(s, amax, float(t.attn_clip), p, ops.new_dropout_seed(dev) if p > 0 else 0, t._diag)
        t.attention_scores = s if t.keep_attn_scores else None
        if t.training:
            t.call_count += 1
        u = ops.attn_pv(probs, in_feat, 1, tag="insq", round_out=not x3)               # P1 h            [B,1,A,C]
        ot = t.out_trans
        z = ops.linear(u[:, 0], ot.first_linear.weight, tag=st, round_out=False)       # (P1 h) Wv^T     [B,A,C]
        # the updated attractors feed the squeeze-out key projection and the value bank (same precision class)
        return ops.layer_norm(z, ot.first_norm_layer.weight, ot.first_norm_layer.bias, consumer_tag=st)

    def forward(self, in_feat, pos_biases=None):
        if pos_biases is not None:
            _unsupported("positional biases with squeezed attention")
        t = self.in_ator_trans
        if t.num_modes == 1 and not t.out_trans.has_FFN and t.out_trans.first_linear.bias is None \
                and t.feat_dim == self.in_feat_dim:
            att = self._in_squeeze_reassociated(in_feat)
        else:
            att = t(self.attractors, in_feat)       # attractors are batch-invariant: projected once
        ops.grad_ready(att, self.ator_out_trans.parameters())       # backward past `att`: the squeeze-out weights are final
        out = self.ator_out_trans(in_feat, att)
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


class SegtranPosEncoder(nn.Module):
    """pos / pos.max() -> learnable sinusoid code; cached in eval mode (reference :1177-1238)."""

    def __init__(self, config):
        super().__init__()
        self.feat_dim = config.trans_in_dim
        self.pos_embed_dim = self.feat_dim
        self.pos_code_type = config.pos_code_type
        if self.pos_code_type != 'lsinu':
            _unsupported("pos_code_type=%r" % self.pos_code_type)
        self.pos_coder = LearnedSinuPosEmbedder(config.pos_dim, self.pos_embed_dim, omega=1, affine=False)
        self.cached_pos_code = None
        self.cached_feat_shape = None

    def forward(self, orig_feat_shape, voxels_pos):
        """voxels_pos [B,N,pd] -> code [N,C0] when the batch shares one set of positions (stride-0 batch dim or
        B == 1), else [B,N,C0].  The global max of the whole tensor normalises the positions (:1231)."""
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
        if self.use_mince_transformer:
            _unsupported("the mince transformer")
        if self.pos_code_type == 'bias':
            print("Squeezed transformer cannot use Positional Biases.")
            print("Please specify '--nosqueeze' to disable squeezed transformer.")
            exit(0)
        self.pos_code_weight = config.pos_code_weight
        self.num_scales = 0
        self.pos_code_layer = SegtranPosEncoder(config)
        layer_cls = SqueezedAttFeatTrans if self.use_squeezed_transformer else CrossAttFeatTrans
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
        for i, layer in enumerate(self.translayers):
            pe = self.pos_code_layer(orig_feat_shape, voxels_pos)
            ln = self.vfeat_norm_layers[i]
            p = self.dropout.p if (self.training and i == 0) else 0.0
            h = ops.prologue(x, ln.weight, ln.bias, pe, float(self.pos_code_weight), mask, p,
                             ops.new_dropout_seed(x.device) if p > 0 else 0)
            ops.grad_ready(h, layer.parameters())                   # backward past `h`: this layer's weights are final
            x = layer(h, pos_biases=None)
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
