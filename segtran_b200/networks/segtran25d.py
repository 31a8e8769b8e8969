"""Segtran25d shell on the H100 hot path — same module surface as the reference's code/networks/segtran25d.py.

The 2.5-D model runs a 2-D backbone (ResNet / EfficientNet) on every depth slice of a [B,C,H,W,D] volume and fuses the
slices' features with one 3-D Squeeze-and-Expansion stack.  The reference permutes every pyramid level into [B,C,H,W,D]
for Conv3d + GroupNorm and builds the full out-FPN map before its class conv; here every feature map stays slice-major,
[B*D2, C, h, w] with slice b*D2 + d, as the backbone emits it:
  * in-FPN: the 2-D pyramid per slice (its GroupNorm is 2-D in the reference too), the bridge conv, then the depth pooling
    D2 -> D3 = D2 // D_pool_K (sx_resize_axis along the slice axis) and one sx_transpose to the reference's (h, w, d)
    token order.
  * out-FPN: Conv3d 1x1x1 is a per-slice GEMM and the depth-preserving trilinear upsampling is bilinear per slice, so each
    stage is ops.fpn_stage(slices=D2); its GroupNorm takes the statistics of a sample over all D2 slices
    (sx_groupnorm_slices_fwd/bwd).  Without the fused path (BatchNorm, unaligned pitches, fusion off) the stock modules
    run on a permuted [B,C,h,w,D2] view.
  * head: the collapsed form (ops.seg_head_slices) — the bridged out-FPN map is never built; with out_fpn_layers ==
    in_fpn_layers the ConvTranspose3d (2,2,1) direct head (ops.direct_head(token_order='hwd')).  Training with
    ``--outdrop`` runs the dropout head on the slice-major map (ops.seg_head_slices_dropout, csrc/sx_head_drop.cu): the
    dropped, depth-upsampled map is never written.  With out_fpn_layers == in_fpn_layers ``--outdrop`` does nothing, as
    in the reference.

Deliberate deviations from the reference:
  * the fusion encoder is called with orig_feat_shape = (H2, W2, D3); the reference passes three arguments to a
    four-argument forward (segtran25d.py:457) and cannot run;
  * positions and scales are built on the input's device, not a 'cuda' literal (:448);
  * an input size that is not an integer multiple of the token grid raises ValueError instead of breakpoint() (:436-437);
  * the ``--outdrop`` mask comes from the library's counter-based generator (seeded per call on the device), so
    ``torch.manual_seed`` does not select it; training with ``--outdrop`` on host tensors raises NotImplementedError
    before any work (the dropout head is CUDA only).
``out_fpn_upsampleD_scheme`` follows the reference's branches (:355-371): 'conv' unfolds depth, 'interpolate' is linear
x D_pool_K, and any other value, including the drivers' default 'interp', leaves the depth at D2.
"""
from __future__ import annotations

from argparse import Namespace

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .segtran2d import Segtran2d, _reference_backbone2d
from .segtran_shared import (CrossAttFeatTrans, ExpandedFeatTrans, SegtranConfig, SegtranFusionEncoder,
                             SegtranInitWeights, bb2feat_dims, gen_all_indices)


class Segtran25dConfig(SegtranConfig):
    """2.5-D application settings (reference segtran25d.py:15-74); attribute names and defaults kept."""

    def __init__(self):
        super().__init__()
        self.backbone_type = 'eff-b3'
        self.use_pretrained = True
        self.bb_feat_dims = bb2feat_dims[self.backbone_type]
        self.num_translayers = 1
        self.set_fpn_layers('default', Namespace(in_fpn_layers='34', out_fpn_layers='1234', in_fpn_scheme='AN',
                                                 out_fpn_scheme='AN', translayer_compress_ratios=[1, 1]),
                            do_print=False)
        self.bb_feat_upsize = True
        self.in_fpn_use_bn = False
        self.out_fpn_use_bn = False
        self.resnet_bn_to_gn = False
        self.G = 8
        self.pos_dim = 3
        self.max_pos_size = (20, 20, 20)          # --pos bias table extent (the 3-D default)
        self.pos_code_every_layer = True          # read by the reference shell (segtran25d.py:92), never used
        self.input_scale = (1., 1., 1.)
        self.num_classes = 2
        self.num_attractors = 1024
        self.orig_in_channels = 1
        self.inchan_to3_scheme = 'stemconv'
        self.D_groupsize = 1
        self.D_pool_K = 2
        self.out_fpn_upsampleD_scheme = 'conv'
        self.device = 'cuda'

    def update_config(self, args):
        self.try_assign(args, 'num_classes', 'backbone_type', 'use_pretrained', 'bb_feat_upsize',
                        'in_fpn_use_bn', 'use_squeezed_transformer', 'num_attractors', 'num_translayers',
                        'num_modes', 'trans_output_type', 'mid_type',
                        'base_initializer_range', 'pos_code_type', 'pos_code_weight', 'pos_bias_radius',
                        'ablate_multihead', 'out_fpn_do_dropout', 'has_FFN_in_squeeze', 'attn_clip',
                        'qk_have_bias', 'tie_qk_scheme', 'orig_in_channels', 'inchan_to3_scheme',
                        'D_groupsize', 'D_pool_K', 'out_fpn_upsampleD_scheme', 'input_scale',
                        'device', 'eval_robustness',
                        'use_mince_transformer', 'mince_scales', 'mince_channel_props')
        if 'dropout_prob' in args and args.dropout_prob >= 0:
            self.hidden_dropout_prob = args.dropout_prob
            self.attention_probs_dropout_prob = args.dropout_prob
            print("Dropout prob: %.2f" % (args.dropout_prob))
        self.bb_feat_dims = bb2feat_dims[self.backbone_type]
        self.set_fpn_layers('args', args)


CONFIG = Segtran25dConfig()


def _to_volume(x, B, D):
    """[B*D, C, h, w] slice-major -> [B, C, h, w, D] (a view)."""
    return x.reshape(B, D, *x.shape[1:]).permute(0, 2, 3, 4, 1)


def _to_slices(x):
    """[B, C, h, w, D] -> [B*D, C, h, w] slice-major."""
    B, C, h, w, D = x.shape
    return x.permute(0, 4, 1, 2, 3).reshape(B * D, C, h, w)


class Segtran25d(SegtranInitWeights):
    def __init__(self, config, backbone=None):
        super().__init__(config)
        self.config = config
        self.device = config.device
        self.orig_in_channels = config.orig_in_channels
        self.trans_in_dim, self.trans_out_dim = config.trans_in_dim, config.trans_out_dim
        self.num_translayers = config.num_translayers
        self.bb_feat_upsize = config.bb_feat_upsize
        self.G = config.G
        self.voxel_fusion = SegtranFusionEncoder(config, 'Fusion')
        self.backbone_type, self.use_pretrained = config.backbone_type, config.use_pretrained
        self.pos_code_every_layer = getattr(config, 'pos_code_every_layer', True)
        own_backbone = backbone is None
        self.backbone = _reference_backbone2d(self.backbone_type, self.use_pretrained, self.bb_feat_upsize) \
            if own_backbone else backbone
        self.inchan_to3_scheme, self.D_groupsize = config.inchan_to3_scheme, config.D_groupsize
        self.eff_in_channels = self.orig_in_channels * self.D_groupsize
        self.D_pool_K = config.D_pool_K
        self.out_fpn_upsampleD_scheme = config.out_fpn_upsampleD_scheme
        self.input_scale = config.input_scale

        if self.eff_in_channels != 3:
            if self.inchan_to3_scheme == 'avgto3':
                if self.eff_in_channels not in (2, 4):
                    raise NotImplementedError("'avgto3' is only for effective channels == 2 or 4, not {}".format(
                        self.eff_in_channels))
                self.in_bridge_to3 = nn.Linear(self.eff_in_channels, 3, bias=False)
                w = [[1, 0], [0.5, 0.5], [0, 1]] if self.eff_in_channels == 2 else \
                    [[1, 0, 0, 0], [0, 0.5, 0.5, 0], [0, 0, 0, 1]]
                self.in_bridge_to3.weight.data.copy_(torch.tensor(w))
                self.in_bridge_to3.weight.requires_grad = False
            elif self.eff_in_channels == 1 and self.inchan_to3_scheme == 'dup3':
                self.in_bridge_to3 = lambda x: x.expand(-1, 3, -1, -1, -1)
            elif self.inchan_to3_scheme == 'bridgeconv':
                self.in_bridge_to3 = nn.Conv3d(self.eff_in_channels, 3, 1)
            elif self.eff_in_channels > 3 and self.inchan_to3_scheme == 'stemconv':
                if not self.backbone_type.startswith('eff'):
                    raise NotImplementedError("Changing stemconv channel number is not supported for {}".format(
                        self.backbone_type))
                if own_backbone:                  # a backbone passed in already takes the 4-channel slices
                    self.backbone._change_in_channels(4, keep_RGB_weight=True)
                self.in_bridge_to3 = nn.Identity()
            else:
                raise NotImplementedError("Effective input channel size={}*{} is not supported for scheme '{}'".format(
                    self.orig_in_channels, self.D_groupsize, self.inchan_to3_scheme))

        self.in_fpn_use_bn, self.in_fpn_layers, self.in_fpn_scheme = \
            config.in_fpn_use_bn, config.in_fpn_layers, config.in_fpn_scheme
        pool_stride = 2 ** int(np.min(self.in_fpn_layers))
        if not self.bb_feat_upsize:
            pool_stride *= 2
        self.mask_pool = nn.AvgPool2d((pool_stride, pool_stride))
        d = self.bb_feat_dims = config.bb_feat_dims
        self.in_fpn23_conv = nn.Conv2d(d[2], d[3], 1)
        self.in_fpn34_conv = nn.Conv2d(d[3], d[4], 1)
        last_in = self.in_fpn_layers[-1]
        self.in_fpn_bridgeconv = nn.Conv2d(d[last_in], self.trans_in_dim, 1) if d[last_in] != self.trans_in_dim \
            else nn.Identity()
        if self.in_fpn_use_bn:
            self.in_bn3b, self.in_bn4b = nn.BatchNorm2d(d[3]), nn.BatchNorm2d(d[4])
            self.in_fpn_norms = [None, None, None, self.in_bn3b, self.in_bn4b]
        else:
            self.in_gn3b, self.in_gn4b = nn.GroupNorm(self.G, d[3]), nn.GroupNorm(self.G, d[4])
            self.in_fpn_norms = [None, None, None, self.in_gn3b, self.in_gn4b]
        self.in_fpn_convs = [None, None, self.in_fpn23_conv, self.in_fpn34_conv]

        self.num_classes = config.num_classes
        self.out_fpn_use_bn, self.out_fpn_layers, self.out_fpn_scheme = \
            config.out_fpn_use_bn, config.out_fpn_layers, config.out_fpn_scheme
        self.out_fpn_do_dropout = config.out_fpn_do_dropout
        self.do_out_fpn = self.out_fpn_layers != self.in_fpn_layers
        if self.do_out_fpn:
            self.out_fpn12_conv3d = nn.Conv3d(d[1], d[2], 1)
            self.out_fpn23_conv3d = nn.Conv3d(d[2], d[3], 1)
            self.out_fpn34_conv3d = nn.Conv3d(d[3], d[4], 1)
            last_out = self.out_fpn_layers[-len(self.in_fpn_layers)]
            self.out_fpn_bridgeconv3d = nn.Conv3d(d[last_out], self.trans_out_dim, 1)
            if self.out_fpn_upsampleD_scheme == 'conv':
                self.out_feat_dim = self.trans_out_dim // self.D_pool_K
                self.out_fpn_upsampleD = nn.Conv3d(self.trans_out_dim, self.out_feat_dim * self.D_pool_K, 1)
            else:
                self.out_feat_dim = self.trans_out_dim
            if self.out_fpn_use_bn:
                self.out_bn2b, self.out_bn3b, self.out_bn4b = \
                    nn.BatchNorm3d(d[2]), nn.BatchNorm3d(d[3]), nn.BatchNorm3d(d[4])
                self.out_fpn_norms = [None, None, self.out_bn2b, self.out_bn3b, self.out_bn4b]
            else:
                self.out_gn2b, self.out_gn3b, self.out_gn4b = \
                    nn.GroupNorm(self.G, d[2]), nn.GroupNorm(self.G, d[3]), nn.GroupNorm(self.G, d[4])
                self.out_fpn_norms = [None, None, self.out_gn2b, self.out_gn3b, self.out_gn4b]
            self.out_fpn_convs = [None, self.out_fpn12_conv3d, self.out_fpn23_conv3d, self.out_fpn34_conv3d]
            self.out_conv3d = nn.Conv3d(self.out_feat_dim, self.num_classes, 1)
            self.out_fpn_dropout = nn.Dropout(config.hidden_dropout_prob)
        else:
            # The reference's 1x1x1 branch tests `'2' in self.in_fpn_layers` on a list of ints, which is never true
            # (as in segtran2d), so every direct head is the ConvTranspose3d.
            self.out_conv3d = nn.ConvTranspose3d(self.trans_out_dim, self.num_classes, (2, 2, 1), (2, 2, 1))

        self.apply(self.init_weights)
        self.apply(self.tie_qk)
        self.apply(self.add_identity_bias)
        self.scales_printed = False
        self.translayer_dims = config.translayer_dims
        self.num_vis_layers = 1 + 2 * self.num_translayers

    def tie_qk(self, module):
        if isinstance(module, CrossAttFeatTrans) and module.tie_qk_scheme != 'none':
            module.tie_qk()

    def add_identity_bias(self, module):
        if isinstance(module, (CrossAttFeatTrans, ExpandedFeatTrans)):
            module.add_identity_bias()

    def get_mask(self, fake2D_batch):
        with torch.no_grad():
            return (self.mask_pool(fake2D_batch.abs()).sum(dim=1) > 0).long()

    def _backbone_feats(self, x):
        if self.backbone_type.startswith('res'):
            return tuple(self.backbone.ext_features(x))
        f = self.backbone.extract_endpoints(x)
        return tuple(f['reduction_%d' % i] for i in range(1, 6))

    def in_fpn_forward(self, batch_base_feats):
        """In-FPN pyramid per slice + bridge conv (reference segtran25d.py:264-288): -> [B*D2, C0, H2, W2]."""
        cur = Segtran2d._pyramid(batch_base_feats, self.in_fpn_layers[:-1], self.in_fpn_convs, self.in_fpn_norms,
                                 self.in_fpn_scheme, self.in_fpn_layers[0])
        bc = self.in_fpn_bridgeconv
        if isinstance(bc, nn.Conv2d) and ops.conv1x1_ok(cur, bc) and ops.fpn_fusion_enabled():
            return ops.conv1x1_add(cur, bc.weight, bc.bias)
        return bc(cur)

    def out_fpn_pyramid(self, batch_base_feats, B, D2):
        """Out-FPN pyramid on slice-major maps (reference segtran25d.py:317-347): -> curr_feat [B*D2, Cf, H1, W1]."""
        cur = batch_base_feats[self.out_fpn_layers[0]]
        for layer in self.out_fpn_layers[:-len(self.in_fpn_layers)]:
            conv, norm = self.out_fpn_convs[layer], self.out_fpn_norms[layer + 1]
            hi = batch_base_feats[layer + 1]
            if isinstance(norm, nn.GroupNorm) and ops.conv1x1_ok(cur, conv) and ops.fpn_fusion_enabled():
                cur = ops.fpn_stage(cur, hi, conv, norm, self.out_fpn_scheme, slices=D2)
                continue
            up = conv(_to_volume(cur, B, D2))
            hi = F.interpolate(_to_volume(hi, B, D2), size=up.shape[2:], mode='trilinear', align_corners=False)
            cur = _to_slices(norm(up + hi) if self.out_fpn_scheme == 'AN' else norm(up) + hi)
        return cur

    def hot_path(self, feat_fpn, curr_feat, vmask, out_size):
        """The CUDA segment of the forward: depth pooling + token flatten -> Squeeze-and-Expansion stack -> collapsed
        voxel-wise head (reference segtran25d.py:290-315, :351-377, :425-477 minus the FPN pyramids).
        feat_fpn [B, D2, C0, H2, W2] (the slice-major in-FPN output viewed per sample); curr_feat [B*D2, Cf, H1, W1]
        (ignored, may be None, without the out-FPN); vmask [B, D2, H2, W2] per-slice mask or None; out_size = (H,W,D)."""
        B, D2, C0, H2, W2 = feat_fpn.shape
        H, W, D = out_size
        D3 = D2 // self.D_pool_K
        grid = torch.Size((H2, W2, D3))
        sH, sW, sD = H // H2, W // W2, D // max(D3, 1)
        if D3 < 1 or sH * H2 != H or sW * W2 != W or sD * D3 != D:
            raise ValueError("input size %s is not an integer multiple of the token grid %s" % ((H, W, D), tuple(grid)))
        drop = self.do_out_fpn and self.out_fpn_do_dropout and self.training
        if drop and not feat_fpn.is_cuda:                     # checked before any work: the head has no host version
            raise NotImplementedError("segtran_b200: --outdrop (out_fpn_do_dropout) in training runs on the CUDA "
                                      "dropout head (csrc/sx_head_drop.cu) only; got %s tensors" % feat_fpn.device)
        HW, X = H2 * W2, C0 * H2 * W2
        # depth pooling on the [B, D2, C0*H2*W2] view, then [B, D3*C0, H2*W2] -> [B, H2*W2, D3*C0] = tokens in (h,w,d)
        pooled = ops.resize_linear(feat_fpn.reshape(B, D2, X), (D3, X))
        vfeat = ops.transpose(pooled.view(B, D3 * C0, HW)).view(B, HW * D3, C0)
        if vmask is not None:
            with torch.no_grad():
                m = ops.resize_linear(vmask.float().reshape(B, D2, HW), (D3, HW)) >= 0.5
                vmask = m.transpose(1, 2).reshape(B, -1).long()
        scale = [sH / self.input_scale[0], sW / self.input_scale[1], sD / self.input_scale[2]]
        if not self.scales_printed:
            print("\nVoxels: %s. Model HWD scales: %dx%dx%d. Total scales: %s" % (list(vfeat.shape), sH, sW, sD, scale))
            self.scales_printed = True
        key = (tuple(grid), tuple(scale), str(vfeat.device))
        if getattr(self, "_pos_cache_key", None) != key:             # built once per shape: no H2D copy per step
            idx = gen_all_indices(grid, device=vfeat.device).view(-1, 3).float() * \
                torch.tensor([scale], device=vfeat.device)
            self._pos_cache_key, self._pos_cache = key, idx
        voxels_pos = self._pos_cache.unsqueeze(0).expand(B, -1, -1)
        fused = self.voxel_fusion(vfeat, voxels_pos, None if vmask is None else vmask.unsqueeze(2), grid)
        head_params = list(self.out_conv3d.parameters())
        unfold = self.do_out_fpn and self.D_pool_K > 1 and self.out_fpn_upsampleD_scheme == 'conv'
        if self.do_out_fpn:
            head_params += list(self.out_fpn_bridgeconv3d.parameters())
        if unfold:
            head_params += list(self.out_fpn_upsampleD.parameters())
        ops.grad_ready(fused, head_params)                            # backward past the head
        self.layers_attn_scores = self.voxel_fusion.layers_attn_scores
        self.orig_feat_shape = grid
        if not self.do_out_fpn:
            return ops.direct_head(fused, tuple(grid), self.out_conv3d.weight, self.out_conv3d.bias, out_size,
                                   token_order='hwd')
        bridge, cls = self.out_fpn_bridgeconv3d, self.out_conv3d
        if drop:                                              # per-channel mask: the dropout head (sx_head_drop.cu)
            ud = self.out_fpn_upsampleD if unfold else None
            return ops.seg_head_slices_dropout(curr_feat, fused, tuple(grid), bridge.weight, bridge.bias, cls.weight,
                                               cls.bias, out_size, self.out_fpn_dropout.p, self.D_pool_K,
                                               self.out_fpn_upsampleD_scheme, Wu=None if ud is None else ud.weight,
                                               bu=None if ud is None else ud.bias)
        if unfold:
            ud = self.out_fpn_upsampleD
            Wc, bc = ops.fold_unfold(cls.weight, cls.bias, ud.weight, ud.bias, self.D_pool_K)
            return ops.seg_head_slices(curr_feat, fused, tuple(grid), bridge.weight, bridge.bias, Wc, bc, out_size,
                                       d_unfold=self.D_pool_K)
        dk = self.D_pool_K if (self.D_pool_K > 1 and self.out_fpn_upsampleD_scheme == 'interpolate') else 1
        return ops.seg_head_slices(curr_feat, fused, tuple(grid), bridge.weight, bridge.bias, cls.weight, cls.bias,
                                   out_size, d_pool_k=dk)

    def forward(self, batch):
        B, C, H, W, D = batch.shape
        assert C == self.orig_in_channels
        if self.D_groupsize > 1:
            g = self.D_groupsize
            batch = batch.view(B, C, H, W, -1, g).permute(0, 1, 5, 2, 3, 4).reshape(B, C * g, H, W, -1)
        D2 = batch.shape[-1]
        x = self.in_bridge_to3(batch) if self.eff_in_channels != 3 else batch
        fake2D_batch = x.permute(0, 4, 1, 2, 3).reshape((-1,) + tuple(x.shape[1:4]))   # [B*D2, C', H, W]
        nonzero_mask = self.get_mask(fake2D_batch)
        feats = self._backbone_feats(fake2D_batch)
        feat_fpn = self.in_fpn_forward(feats)
        curr_feat = self.out_fpn_pyramid(feats, B, D2) if self.do_out_fpn else None
        vmask = nonzero_mask.view(B, D2, *nonzero_mask.shape[1:])
        return self.hot_path(feat_fpn.view(B, D2, *feat_fpn.shape[1:]), curr_feat, vmask, (H, W, D))
