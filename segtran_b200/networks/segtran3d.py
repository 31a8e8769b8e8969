"""Segtran3d shell on the H100 hot path — same module surface as the reference's code/networks/segtran3d.py.

What runs where
  * CNN backbone (I3D) and the in-/out-FPN pyramids (1x1x1 conv + trilinear + GroupNorm): stock PyTorch/cuDNN
    (out of the hot path, SURVEY.md §8f "next").  The backbone class is the reference's own
    ``networks.aj_i3d.aj_i3d.InceptionI3d`` when this package is dropped into the reference tree, or any module
    with ``extract_features`` passed as ``backbone=``.
  * token flatten, Squeeze-and-Expansion stack, scatter and the voxel-wise head: segtran_b200 kernels.
    The head uses the collapsed form (csrc/sx_head.cu): ``out_fpn_bridgeconv3d`` and ``out_conv3d`` keep their
    own parameters (checkpoint compatible) but are applied as one class-dimension contraction.  ``--upd conv``
    (``out_fpn_upsampleD``) is linear too and is folded into the class conv in weight space.  ``--outdrop`` in training
    runs the dropout head (csrc/sx_head_drop.cu), which never writes the dropped full-resolution map.
    With out_fpn_layers == in_fpn_layers there is no out-FPN: ``out_conv3d`` is a ConvTranspose3d on the tokens, run
    with the trilinear interpolation as ``ops.direct_head``.
"""
from __future__ import annotations

import os
from argparse import Namespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from .segtran_shared import (CrossAttFeatTrans, ExpandedFeatTrans, SegtranConfig, SegtranFusionEncoder,
                             SegtranInitWeights, bb2feat_dims, gen_all_indices)


class Segtran3dConfig(SegtranConfig):
    """3-D application settings (reference segtran3d.py:19-77); attribute names and defaults kept."""

    def __init__(self):
        super().__init__()
        self.backbone_type = 'i3d'
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
        self.max_pos_size = (20, 20, 20)
        self.input_scale = (1., 1., 1.)
        self.num_classes = 2
        self.num_attractors = 1024
        self.orig_in_channels = 1
        self.inchan_to3_scheme = 'bridgeconv'
        self.D_groupsize = 1
        self.D_pool_K = 2
        self.out_fpn_upsampleD_scheme = 'interp'
        self.device = 'cuda'

    def update_config(self, args):
        self.try_assign(args, 'num_classes', 'backbone_type', 'use_pretrained', 'bb_feat_upsize', 'in_fpn_use_bn',
                        'use_squeezed_transformer', 'num_attractors', 'num_translayers', 'num_modes',
                        'trans_output_type', 'mid_type', 'pos_code_type', 'pos_code_weight', 'pos_bias_radius',
                        'ablate_multihead', 'out_fpn_do_dropout', 'has_FFN_in_squeeze', 'attn_clip', 'qk_have_bias',
                        'tie_qk_scheme', 'orig_in_channels', 'inchan_to3_scheme', 'D_groupsize', 'D_pool_K',
                        'out_fpn_upsampleD_scheme', 'input_scale', 'device', 'eval_robustness',
                        'use_attn_consist_loss', 'use_mince_transformer', 'mince_scales', 'mince_channel_props')
        if 'dropout_prob' in args and args.dropout_prob >= 0:
            self.hidden_dropout_prob = args.dropout_prob
            self.attention_probs_dropout_prob = args.dropout_prob
            print("Dropout prob: %.2f" % (args.dropout_prob))
        self.bb_feat_dims = bb2feat_dims[self.backbone_type]
        self.set_fpn_layers('args', args)


CONFIG = Segtran3dConfig()

_I3D_KEYS = ('MaxPool3d_2a_3x3', 'Conv3d_2c_3x3', 'Mixed_3c', 'Mixed_4f', 'Mixed_5c')


def _reference_i3d(do_pool1, use_pretrained):
    """The backbone is out of scope for this package: take the reference's InceptionI3d when it is importable
    (i.e. when segtran_b200 is used as a drop-in inside the reference tree)."""
    try:
        import networks.aj_i3d.aj_i3d as aj_i3d
    except Exception as e:                                   # noqa: BLE001
        raise RuntimeError(
            "Segtran3d needs an I3D backbone: put the reference's code/ directory on sys.path (drop-in use) or "
            "pass backbone=<module with extract_features()> to Segtran3d(...)") from e
    net = aj_i3d.InceptionI3d(do_pool1=do_pool1)
    if use_pretrained:
        path = os.path.join(os.path.dirname(aj_i3d.__file__), "aj_rgb_imagenet.pth")
        net.load_state_dict(torch.load(path, map_location='cpu'))
        print("Loaded pretrained i3d model '{}'".format(path))
    return net


class Segtran3d(SegtranInitWeights):
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
        if not self.backbone_type.startswith('i3d'):
            raise NotImplementedError("Only support i3d as the 3D backbone")
        self.backbone = backbone if backbone is not None else _reference_i3d(not self.bb_feat_upsize,
                                                                             self.use_pretrained)
        self.inchan_to3_scheme, self.D_groupsize = config.inchan_to3_scheme, config.D_groupsize
        self.eff_in_channels = self.orig_in_channels * self.D_groupsize
        self.D_pool_K = config.D_pool_K
        self.out_fpn_upsampleD_scheme = config.out_fpn_upsampleD_scheme
        self.input_scale = config.input_scale
        if self.out_fpn_upsampleD_scheme not in ('interp', 'none', 'conv'):
            raise NotImplementedError("out_fpn_upsampleD_scheme=%r" % self.out_fpn_upsampleD_scheme)

        if self.eff_in_channels != 3:
            if self.inchan_to3_scheme == 'avgto3' and self.eff_in_channels in (2, 4):
                self.in_bridge_to3 = nn.Linear(self.eff_in_channels, 3, bias=False)
                w = [[1, 0], [0.5, 0.5], [0, 1]] if self.eff_in_channels == 2 else \
                    [[1, 0, 0, 0], [0, 0.5, 0.5, 0], [0, 0, 0, 1]]
                self.in_bridge_to3.weight.data.copy_(torch.tensor(w))
                self.in_bridge_to3.weight.requires_grad = False
            elif self.eff_in_channels == 1 and self.inchan_to3_scheme == 'dup3':
                self.in_bridge_to3 = lambda x: x.expand(-1, 3, -1, -1, -1)
            elif self.inchan_to3_scheme == 'bridgeconv':
                self.in_bridge_to3 = nn.Conv3d(self.eff_in_channels, 3, 1)
            else:
                raise NotImplementedError("Effective input channel size={}*{} is not supported for scheme '{}'".format(
                    self.orig_in_channels, self.D_groupsize, self.inchan_to3_scheme))

        self.in_fpn_use_bn, self.in_fpn_layers, self.in_fpn_scheme = \
            config.in_fpn_use_bn, config.in_fpn_layers, config.in_fpn_scheme
        lo = 2 if 2 in self.in_fpn_layers else (3 if 3 in self.in_fpn_layers else 4)
        k = {2: (2, 4, 4), 3: (4, 8, 8), 4: (8, 16, 16)}[lo]
        if not self.bb_feat_upsize:
            k = (k[0], k[1] * 2, k[2] * 2)
        self.mask_pool = nn.AvgPool3d(k)

        d = self.bb_feat_dims = config.bb_feat_dims
        self.in_fpn23_conv = nn.Conv3d(d[2], d[3], 1)
        self.in_fpn34_conv = nn.Conv3d(d[3], d[4], 1)
        last_in = self.in_fpn_layers[-1]
        self.in_fpn_bridgeconv = nn.Conv3d(d[last_in], self.trans_in_dim, 1) if d[last_in] != self.trans_in_dim \
            else nn.Identity()
        if self.in_fpn_use_bn:
            self.in_bn3b, self.in_bn4b = nn.BatchNorm3d(d[3]), nn.BatchNorm3d(d[4])
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
            last_out = self.out_fpn_layers[-len(self.in_fpn_layers)]
            self.out_fpn_out_dim = self.trans_out_dim
            self.out_fpn12_conv3d = nn.Conv3d(d[1], d[2], 1)
            self.out_fpn23_conv3d = nn.Conv3d(d[2], d[3], 1)
            self.out_fpn34_conv3d = nn.Conv3d(d[3], d[4], 1)
            self.out_fpn_bridgeconv3d = nn.Conv3d(d[last_out], self.trans_out_dim, 1)
            if self.out_fpn_upsampleD_scheme == 'conv':
                # created here, before the norms, as the reference does: seeded construction draws the same weights
                self.out_feat_dim = self.out_fpn_out_dim // self.D_pool_K
                self.out_fpn_upsampleD = nn.Conv3d(self.out_fpn_out_dim, self.out_feat_dim * self.D_pool_K, 1)
            else:
                self.out_feat_dim = self.out_fpn_out_dim
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
            # Class scores straight from the tokens, as the 2-D shell does: ConvTranspose3d (2,2,1) on the (H,W,D)-permuted
            # tokens (the reference's 1x1x1-conv branch for '234' is never taken, see segtran2d).  --upd conv and --outdrop
            # have no out-FPN map to act on.
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

    def get_mask(self, batch):
        with torch.no_grad():
            return (self.mask_pool(batch.abs()).sum(dim=1) > 0).long()

    @staticmethod
    def _pyramid(feats, layers, convs, norms, scheme, start):
        """conv1x1(curr) (+) trilinear(higher) -> norm, bottom-up over `layers` (reference segtran3d.py:299-313, :347-359 /
        segtran2d.py:244-257, :286-300).  On CUDA with GroupNorm and TMA-legal shapes each stage is the fused
        ops.fpn_stage (conv + bias + add in one wgmma GEMM, two-pass GroupNorm); otherwise the stock modules run."""
        cur = feats[start]
        for layer in layers:
            conv, norm = convs[layer], norms[layer + 1]
            if isinstance(norm, nn.GroupNorm) and ops.conv1x1_ok(cur, conv) and ops.fpn_fusion_enabled():
                cur = ops.fpn_stage(cur, feats[layer + 1], conv, norm, scheme)
                continue
            up = conv(cur)
            hi = F.interpolate(feats[layer + 1], size=up.shape[2:], mode='trilinear', align_corners=False)
            cur = norm(up + hi) if scheme == 'AN' else norm(up) + hi
        return cur

    def in_fpn_forward(self, batch_base_feats, nonzero_mask):
        """In-FPN pyramid + depth pooling: -> feat_fpn [B,C0,D2,H2,W2], vmask [B,N]."""
        cur = self._pyramid(batch_base_feats, self.in_fpn_layers[:-1], self.in_fpn_convs, self.in_fpn_norms,
                            self.in_fpn_scheme, self.in_fpn_layers[0])
        bc = self.in_fpn_bridgeconv
        if isinstance(bc, nn.Conv3d) and ops.conv1x1_ok(cur, bc) and ops.fpn_fusion_enabled():
            cur = ops.conv1x1_add(cur, bc.weight, bc.bias)               # 1x1x1 bridge conv as one GEMM
        else:
            cur = bc(cur)
        size = list(cur.shape[2:])
        size[0] //= self.D_pool_K
        if ops.fpn_fusion_enabled():                                     # depth pooling / mask pooling: sx_resize_axis
            cur = ops.resize_linear(cur, size)
            m = ops.resize_linear(nonzero_mask.float().unsqueeze(1), size)
        else:
            cur = F.interpolate(cur, size=size, mode='trilinear', align_corners=False)
            m = F.interpolate(nonzero_mask.float().unsqueeze(1), size=size, mode='trilinear', align_corners=False)
        vmask = (m.squeeze(1) >= 0.5).long().reshape(cur.shape[0], -1)
        return cur, vmask

    def out_fpn_pyramid(self, batch_base_feats):
        """Out-FPN pyramid (stock ops): -> curr_feat [B,Cf,D1,H1,W1], the head's dense input."""
        layers = self.out_fpn_layers[:-len(self.in_fpn_layers)]
        return self._pyramid(batch_base_feats, layers, self.out_fpn_convs, self.out_fpn_norms, self.out_fpn_scheme,
                             self.out_fpn_layers[0])

    def hot_path(self, feat_fpn, curr_feat, vmask, out_size):
        """The CUDA segment of the forward: token flatten -> Squeeze-and-Expansion stack -> scatter -> collapsed
        voxel-wise head (reference segtran3d.py:326-332, :442-498 minus the FPN pyramids).
        feat_fpn [B,C0,D2,H2,W2], curr_feat [B,Cf,D1,H1,W1] (ignored, may be None, without the out-FPN), vmask [B,N] or
        None, out_size = (H,W,D) -> logits."""
        B, C0, D2, H2, W2 = feat_fpn.shape
        H, W, D = out_size
        grid = torch.Size((D2, H2, W2))
        sH, sW, sD = H // H2, W // W2, D // D2                        # D: depth of the original volume (reference :446)
        if sH * H2 != H or sW * W2 != W or sD * D2 != D:
            raise ValueError("input size %s is not an integer multiple of the token grid %s" % ((H, W, D), tuple(grid)))
        vfeat = ops.transpose(feat_fpn.reshape(B, C0, -1))            # [B,C0,N] -> [B,N,C0]  (flatten kernel)
        scale = [sD / self.input_scale[2], sH / self.input_scale[0], sW / self.input_scale[1]]
        if not self.scales_printed:
            print("\nFeat: %s, Voxels: %s. Model DHW scales: %dx%dx%d. Total scales: %s" %
                  (list(grid), list(vfeat.shape), sD, sH, sW, scale))
            self.scales_printed = True
        key = (tuple(grid), tuple(scale), str(vfeat.device))
        if getattr(self, "_pos_cache_key", None) != key:             # built once per shape: no H2D copy per step
            idx = gen_all_indices(grid, device=vfeat.device).view(-1, 3).float() * \
                torch.tensor([scale], device=vfeat.device)
            self._pos_cache_key, self._pos_cache = key, idx
        voxels_pos = self._pos_cache.unsqueeze(0).expand(B, -1, -1)  # one set of positions, shared by the batch
        fused = self.voxel_fusion(vfeat, voxels_pos, None if vmask is None else vmask.unsqueeze(2), grid)
        head_params = list(self.out_conv3d.parameters())
        if self.do_out_fpn:
            head_params += list(self.out_fpn_bridgeconv3d.parameters())
        if self.do_out_fpn and self.out_fpn_upsampleD_scheme == 'conv':
            head_params += list(self.out_fpn_upsampleD.parameters())
        ops.grad_ready(fused, head_params)                            # backward past the head
        self.layers_attn_scores = self.voxel_fusion.layers_attn_scores
        self.orig_feat_shape = grid
        if not self.do_out_fpn:                 # ConvTranspose3d + trilinear: the direct head (curr_feat unused)
            return ops.direct_head(fused, tuple(grid), self.out_conv3d.weight, self.out_conv3d.bias, out_size)
        bridge, cls = self.out_fpn_bridgeconv3d, self.out_conv3d
        # the depth upsampling runs only when D_pool_K > 1 (reference segtran3d.py:372)
        unfold = self.D_pool_K > 1 and self.out_fpn_upsampleD_scheme == 'conv'
        if self.out_fpn_do_dropout and self.training:
            ud = self.out_fpn_upsampleD if unfold else None
            return ops.seg_head_dropout(curr_feat, fused, tuple(grid), bridge.weight, bridge.bias, cls.weight, cls.bias,
                                        out_size, self.out_fpn_dropout.p, d_pool_k=self.D_pool_K,
                                        upsample_d=self.out_fpn_upsampleD_scheme,
                                        Wu=None if ud is None else ud.weight, bu=None if ud is None else ud.bias)
        if unfold:
            ud = self.out_fpn_upsampleD
            Wf, bf = ops.fold_unfold(cls.weight, cls.bias, ud.weight, ud.bias, self.D_pool_K)
            return ops.seg_head(curr_feat, fused, tuple(grid), bridge.weight, bridge.bias, Wf, bf, out_size,
                                d_unfold=self.D_pool_K)
        dk = self.D_pool_K if (self.D_pool_K > 1 and self.out_fpn_upsampleD_scheme == 'interp') else 1
        return ops.seg_head(curr_feat, fused, tuple(grid), self.out_fpn_bridgeconv3d.weight,
                            self.out_fpn_bridgeconv3d.bias, self.out_conv3d.weight, self.out_conv3d.bias, out_size,
                            d_pool_k=dk)

    def forward(self, batch):
        B, C, H, W, D = batch.shape
        assert C == self.orig_in_channels
        if self.D_groupsize > 1:
            g = self.D_groupsize
            batch = batch.view(B, C, H, W, -1, g).permute(0, 1, 5, 2, 3, 4).reshape(B, C * g, H, W, -1)
        x = batch
        if self.eff_in_channels != 3:
            x = self.in_bridge_to3(x)
        x = x.permute(0, 1, 4, 2, 3)                                  # (H,W,D) -> (D,H,W) frames-first for I3D
        nonzero_mask = self.get_mask(x)
        f = self.backbone.extract_features(x)
        feats = tuple(f[k] for k in _I3D_KEYS)
        feat_fpn, vmask = self.in_fpn_forward(feats, nonzero_mask)
        curr_feat = self.out_fpn_pyramid(feats) if self.do_out_fpn else None
        return self.hot_path(feat_fpn, curr_feat, vmask, (H, W, D))
