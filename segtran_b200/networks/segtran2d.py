"""Segtran2d shell on the H100 hot path — same module surface as the reference's code/networks/segtran2d.py.

Backbone (ResNet / EfficientNet) and the in-/out-FPN pyramids stay stock PyTorch/cuDNN (out of the hot path);
token flatten, the Squeeze-and-Expansion stack and the pixel-wise head (collapsed form) run on segtran_b200 kernels.
The backbone is the reference's own class when this package is dropped into the reference tree
(``resnet`` / ``efficientnet.model`` importable), or any module passed as ``backbone=``.
"""
from __future__ import annotations

from argparse import Namespace

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .segtran_shared import (CrossAttFeatTrans, ExpandedFeatTrans, SegtranConfig, SegtranFusionEncoder,
                             SegtranInitWeights, bb2feat_dims, gen_all_indices)


class Segtran2dConfig(SegtranConfig):
    """2-D application settings (reference segtran2d.py:16-63); attribute names and defaults kept."""

    def __init__(self):
        super().__init__()
        self.backbone_type = 'eff-b4'
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
        self.pos_dim = 2
        self.max_pos_size = (100, 100)
        self.num_classes = 2
        self.num_modalities = 0
        self.use_attention_consist_loss = False
        self.use_global_bias = False
        self.device = 'cuda'

    def update_config(self, args):
        self.try_assign(args, 'num_classes', 'backbone_type', 'use_pretrained', 'bb_feat_upsize', 'in_fpn_use_bn',
                        'use_squeezed_transformer', 'num_attractors', 'num_translayers', 'num_modes',
                        'trans_output_type', 'mid_type', 'pos_code_type', 'pos_code_weight', 'pos_bias_radius',
                        'ablate_multihead', 'out_fpn_do_dropout', 'has_FFN_in_squeeze', 'attn_clip', 'qk_have_bias',
                        'tie_qk_scheme', 'num_modalities', 'device', 'eval_robustness', 'use_global_bias',
                        'use_attn_consist_loss', 'use_mince_transformer', 'mince_scales', 'mince_channel_props')
        if 'dropout_prob' in args and args.dropout_prob >= 0:
            self.hidden_dropout_prob = args.dropout_prob
            self.attention_probs_dropout_prob = args.dropout_prob
            print("Dropout prob: %.2f" % (args.dropout_prob))
        self.bb_feat_dims = bb2feat_dims[self.backbone_type]
        self.set_fpn_layers('args', args)


CONFIG = Segtran2dConfig()


def _reference_backbone2d(backbone_type, use_pretrained, bb_feat_upsize):
    """Backbones are out of scope here: use the reference's classes when importable (drop-in use)."""
    try:
        if backbone_type.startswith('res'):
            import resnet
            return resnet.__dict__[backbone_type](pretrained=use_pretrained, do_pool1=not bb_feat_upsize)
        if backbone_type.startswith('eff-'):
            from efficientnet.model import EfficientNet
            name = backbone_type.replace("eff", "efficientnet")
            stem_stride = 1 if bb_feat_upsize else 2
            if use_pretrained:
                return EfficientNet.from_pretrained(name, advprop=True, ignore_missing_keys=True,
                                                    stem_stride=stem_stride)
            return EfficientNet.from_name(name, stem_stride=stem_stride)
    except ImportError as e:
        raise RuntimeError(
            "Segtran2d needs a CNN backbone: put the reference's code/ directory on sys.path (drop-in use) or pass "
            "backbone=<module> to Segtran2d(...)") from e
    raise NotImplementedError("segtran_b200: backbone_type %r (timm EfficientNetV2) must be passed as backbone="
                              % backbone_type)


class Segtran2d(SegtranInitWeights):
    def __init__(self, config, backbone=None):
        super().__init__(config)
        self.config = config
        self.device = config.device
        self.trans_in_dim, self.trans_out_dim = config.trans_in_dim, config.trans_out_dim
        self.num_translayers = config.num_translayers
        self.bb_feat_upsize = config.bb_feat_upsize
        self.G = config.G
        self.use_global_bias = config.use_global_bias
        if self.use_global_bias:
            raise NotImplementedError("segtran_b200: use_global_bias (an ablation without the transformer)")
        self.voxel_fusion = SegtranFusionEncoder(config, 'Fusion')
        self.vfeat_bias = None
        self.vfeat_bias_norm_layer = nn.Identity()
        self.backbone_type, self.use_pretrained = config.backbone_type, config.use_pretrained
        self.backbone = backbone if backbone is not None else _reference_backbone2d(
            self.backbone_type, self.use_pretrained, self.bb_feat_upsize)

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
        self.num_modalities = config.num_modalities
        if self.num_modalities > 0:
            self.mod_fuse_conv = nn.Conv2d(self.num_modalities, 1, 1)
        self.out_fpn_use_bn, self.out_fpn_layers, self.out_fpn_scheme = \
            config.out_fpn_use_bn, config.out_fpn_layers, config.out_fpn_scheme
        self.out_fpn_do_dropout = config.out_fpn_do_dropout
        if self.out_fpn_layers == self.in_fpn_layers:
            raise NotImplementedError("segtran_b200: out_fpn_layers == in_fpn_layers (ConvTranspose2d head) is not "
                                      "implemented; the drivers use in='34', out='1234'")
        self.do_out_fpn = True
        self.out_fpn12_conv = nn.Conv2d(d[1], d[2], 1)
        self.out_fpn23_conv = nn.Conv2d(d[2], d[3], 1)
        self.out_fpn34_conv = nn.Conv2d(d[3], d[4], 1)
        last_out = self.out_fpn_layers[-len(self.in_fpn_layers)]
        self.out_fpn_bridgeconv = nn.Conv2d(d[last_out], self.trans_out_dim, 1) if d[last_out] != self.trans_out_dim \
            else nn.Identity()
        if self.out_fpn_use_bn:
            self.out_bn2b, self.out_bn3b, self.out_bn4b = nn.BatchNorm2d(d[2]), nn.BatchNorm2d(d[3]), nn.BatchNorm2d(d[4])
            self.out_fpn_norms = [None, None, self.out_bn2b, self.out_bn3b, self.out_bn4b]
        else:
            self.out_gn2b, self.out_gn3b, self.out_gn4b = \
                nn.GroupNorm(self.G, d[2]), nn.GroupNorm(self.G, d[3]), nn.GroupNorm(self.G, d[4])
            self.out_fpn_norms = [None, None, self.out_gn2b, self.out_gn3b, self.out_gn4b]
        self.out_fpn_convs = [None, self.out_fpn12_conv, self.out_fpn23_conv, self.out_fpn34_conv]
        self.out_conv = nn.Conv2d(self.trans_out_dim, self.num_classes, 1)
        self.out_fpn_dropout = nn.Dropout(config.hidden_dropout_prob)

        self.apply(self.init_weights)
        self.apply(self.tie_qk)
        self.apply(self.add_identity_bias)
        if self.num_modalities > 0:
            self.mod_fuse_conv.weight.data.fill_(1 / self.num_modalities)
            self.mod_fuse_conv.bias.data.zero_()
        self.scales_printed = False
        self.translayer_dims = config.translayer_dims
        self.num_vis_layers = 1 + 2 * self.num_translayers
        self.feature_maps = []

    def tie_qk(self, module):
        if isinstance(module, CrossAttFeatTrans) and module.tie_qk_scheme != 'none':
            module.tie_qk()

    def add_identity_bias(self, module):
        if isinstance(module, (CrossAttFeatTrans, ExpandedFeatTrans)):
            module.add_identity_bias()

    def get_mask(self, batch):
        with torch.no_grad():
            return self.mask_pool(batch.abs()).sum(dim=1) > 0

    @staticmethod
    def _pyramid(feats, layers, convs, norms, scheme, start):
        """conv1x1(curr) (+) bilinear(higher) -> norm, bottom-up over `layers` (reference segtran3d.py:299-313, :347-359 /
        segtran2d.py:244-257, :286-300).  On CUDA with GroupNorm and TMA-legal shapes each stage is the fused
        ops.fpn_stage (conv + bias + add in one wgmma GEMM, two-pass GroupNorm); otherwise the stock modules run."""
        cur = feats[start]
        for layer in layers:
            conv, norm = convs[layer], norms[layer + 1]
            if isinstance(norm, nn.GroupNorm) and ops.conv1x1_ok(cur, conv) and ops.fpn_fusion_enabled():
                cur = ops.fpn_stage(cur, feats[layer + 1], conv, norm, scheme)
                continue
            up = conv(cur)
            hi = F.interpolate(feats[layer + 1], size=up.shape[2:], mode='bilinear', align_corners=False)
            cur = norm(up + hi) if scheme == 'AN' else norm(up) + hi
        return cur

    def _backbone_feats(self, batch):
        if self.backbone_type.startswith('res'):
            return tuple(self.backbone.ext_features(batch))
        if self.backbone_type.startswith('eff-'):
            f = self.backbone.extract_endpoints(batch)
            return tuple(f['reduction_%d' % i] for i in range(1, 6))
        return tuple(self.backbone(batch))

    def hot_path(self, feat_fpn, curr_feat, vmask, out_size, B0=None, MOD=0):
        """The CUDA segment: token flatten -> Squeeze-and-Expansion stack -> scatter -> collapsed pixel-wise head
        (reference segtran2d.py:264-269, :362-436 minus the FPN pyramids).
        feat_fpn [B,C0,H2,W2], curr_feat [B,Cf,H1,W1], vmask [B,N] or None, out_size = (H,W) -> logits."""
        B, C0, H2, W2 = feat_fpn.shape
        B0 = B if B0 is None else B0
        H, W = out_size
        vfeat = ops.transpose(feat_fpn.reshape(B, C0, -1))                   # [B,C0,N] -> [B,N,C0]
        if MOD > 0:
            vfeat = vfeat.view(B0, MOD, -1, self.trans_in_dim).max(dim=1)[0]
        grid = torch.Size((H2, W2))
        sH, sW = H // H2, W // W2
        if sH * H2 != H or sW * W2 != W:
            raise ValueError("input size %s is not an integer multiple of the token grid %s" % ((H, W), tuple(grid)))
        if not self.scales_printed:
            print("\nImage scales: %dx%d. Feat: %s. Voxels: %s" % (sH, sW, list(grid), list(vfeat.shape)))
            self.scales_printed = True
        key = (tuple(grid), sH, sW, str(vfeat.device))
        if getattr(self, "_pos_cache_key", None) != key:             # built once per shape: no H2D copy per step
            idx = gen_all_indices(grid, device=vfeat.device).view(-1, 2).float() * \
                torch.tensor([[float(sH), float(sW)]], device=vfeat.device)
            self._pos_cache_key, self._pos_cache = key, idx
        voxels_pos = self._pos_cache.unsqueeze(0).expand(B0, -1, -1)
        fused = self.voxel_fusion(vfeat, voxels_pos, None if vmask is None else vmask.unsqueeze(2), grid)
        ops.grad_ready(fused, list(self.out_fpn_bridgeconv.parameters()) + list(self.out_conv.parameters()))   # backward past the head
        self.layers_attn_scores = self.voxel_fusion.layers_attn_scores
        for i in range(self.num_translayers):
            self.feature_maps.append(self.voxel_fusion.translayers[i].attention_scores)
        for i in range(self.num_translayers):
            lv = self.voxel_fusion.layers_vfeat[i]
            self.feature_maps.append(lv.detach().view(B0, H2, W2, self.translayer_dims[i + 1]).permute(0, 3, 1, 2))
        self.orig_feat_shape = grid
        if self.out_fpn_do_dropout and self.training:
            raise NotImplementedError("segtran_b200: out_fpn_do_dropout breaks the linear head collapse")
        bridge = self.out_fpn_bridgeconv
        Wb, bb = (bridge.weight, bridge.bias) if isinstance(bridge, nn.Conv2d) else (None, None)
        return ops.seg_head(curr_feat, fused, tuple(grid), Wb, bb, self.out_conv.weight, self.out_conv.bias, (H, W))

    def forward(self, batch):
        self.feature_maps = []
        MOD = 0
        B0 = batch.shape[0]
        if self.num_modalities > 0:
            B0, C, H, W, MOD = batch.shape
            batch = batch.view(B0 * MOD, C, H, W)                    # as the reference does (segtran2d.py:324-331)
        B, C, H, W = batch.shape
        nonzero_mask = self.get_mask(batch)
        feats = self._backbone_feats(batch)
        cur = self._pyramid(feats, self.in_fpn_layers[:-1], self.in_fpn_convs, self.in_fpn_norms, self.in_fpn_scheme,
                            self.in_fpn_layers[0])
        bc = self.in_fpn_bridgeconv
        if isinstance(bc, nn.Conv2d) and ops.conv1x1_ok(cur, bc) and ops.fpn_fusion_enabled():
            feat_fpn = ops.conv1x1_add(cur, bc.weight, bc.bias)          # 1x1 bridge conv as one GEMM
        else:
            feat_fpn = bc(cur)
        self.feature_maps.append(feat_fpn)
        layers = self.out_fpn_layers[:-len(self.in_fpn_layers)]
        curr_feat = self._pyramid(feats, layers, self.out_fpn_convs, self.out_fpn_norms, self.out_fpn_scheme,
                                  self.out_fpn_layers[0])
        return self.hot_path(feat_fpn, curr_feat, nonzero_mask.reshape(B, -1), (H, W), B0, MOD)
