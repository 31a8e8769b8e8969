"""Generate the tests/golden/seg25d_*.pt fixtures of the 2.5-D model from the REAL reference Segtran25d.

TEST INFRASTRUCTURE ONLY.  Run in the build container:  python -m oracle.gen_seg25d_golden
The reference shell cannot run as it stands, so three things are patched around it, none inside the computation:
  * its config has no ``pos_code_every_layer`` (read at segtran25d.py:92, never used) nor ``max_pos_size`` (read by the
    --pos bias encoder): both are set on the config, max_pos_size to the token grid; --pos bias tables get seeded
    values (they are zero-initialised);
  * ``voxel_fusion.forward`` is called with three arguments (:457): a wrapper passes the (H2, W2, D3) token grid;
  * the ``device='cuda'`` literal (:448) goes to the CPU (ref_import.cuda_literal_to_cpu).
Backbones are stand-ins returning stored per-slice features ([B*D2, C, h, w], feature widths [8, 8, 16, 16, 32]); the
EfficientNet-named one also records the reference's stem change (_change_in_channels(4)).  Volumes are (H,W,D) =
(16,16,8) (D = 16 with D_groupsize 2): token grid (H2, W2, D3) = (2, 2, 4), out-FPN head at 8x8 per slice.
Loss = (out * G).sum(); each fixture stores the seeded input, the state dict without backbone keys, the logits and the
gradients to the parameters and to the features.  Cases:
  seg25d_stemconv   eff stand-in, 4 modalities, stemconv, a zero depth slab (masked tokens), --upd interpolate
  seg25d_updconv    resnet stand-in, 2 modalities, bridgeconv, --upd conv, 3 classes
  seg25d_dgroup2    D_groupsize 2 (bridgeconv), --upd interp (the drivers' default: no depth map in the reference)
  seg25d_direct34   --outfpn 34: the ConvTranspose3d (2,2,1) direct head
  seg25d_posbias    --nosqueeze --pos bias, which reads the (H2, W2, D3) grid in the encoder
"""
from __future__ import annotations

import os
import sys
from argparse import Namespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import as R                                                # noqa: E402
from oracle.gen_golden import OUT, _grads                                        # noqa: E402

DIMS = [8, 8, 16, 16, 32]
H = W = 16


class FixedFeatEff(torch.nn.Module):
    """Stands in for EfficientNet.extract_endpoints (efficientnet/model.py) with stored features."""

    def __init__(self):
        super().__init__()
        self.feats = None
        self.in_channels_changed = None

    def _change_in_channels(self, in_channels, keep_RGB_weight=False):
        self.in_channels_changed = (in_channels, keep_RGB_weight)

    def extract_endpoints(self, x):
        return {'reduction_%d' % (i + 1): f for i, f in enumerate(self.feats)}


class FixedFeatRes(torch.nn.Module):
    """Stands in for ResNet.ext_features (resnet.py:186-200)."""

    def __init__(self):
        super().__init__()
        self.feats = None

    def ext_features(self, x):
        return tuple(self.feats)


def _args(**kw):
    a = dict(num_classes=2, use_pretrained=False, num_attractors=6, num_translayers=1, num_modes=2,
             trans_output_type="private", mid_type="shared", device="cpu", in_fpn_layers="34", out_fpn_layers="1234",
             in_fpn_scheme="AN", out_fpn_scheme="AN", translayer_compress_ratios=[1, 1], dropout_prob=0.0,
             tie_qk_scheme="shared", qk_have_bias=True, use_squeezed_transformer=True, pos_code_type="lsinu",
             out_fpn_do_dropout=False, D_pool_K=2, D_groupsize=1, input_scale=(1., 1., 1.))
    a.update(kw)
    return Namespace(**a)


def gen(name, seed, args, C, D, zero_slab=False):
    ns = R.load()
    import networks.segtran25d as seg25d
    import resnet as ref_resnet
    ns.shared.bb2feat_dims[args.backbone_type] = DIMS
    eff = FixedFeatEff()
    res = FixedFeatRes()
    ref_resnet.__dict__[args.backbone_type] = lambda pretrained=False, do_pool1=True: res
    orig_from_name = seg25d.EfficientNet.from_name
    seg25d.EfficientNet.from_name = classmethod(lambda cls, *a, **k: eff)
    cfg = seg25d.CONFIG
    g = args.D_groupsize
    D2 = D // g
    H2, W2, D3 = H // 8, W // 8, D2 // args.D_pool_K
    cfg.pos_code_every_layer = True
    cfg.max_pos_size = (H2, W2, D3)                     # keeps the reference's --pos bias index buffers small
    torch.manual_seed(seed)
    try:
        with R.quiet():
            cfg.update_config(args)
            net = seg25d.Segtran25d(cfg)
    finally:
        seg25d.EfficientNet.from_name = orig_from_name
    bb = net.backbone
    if args.pos_code_type == "bias":                    # zero-initialised: seeded values so the forward exercises them
        with torch.no_grad():
            net.voxel_fusion.pos_code_layer.pos_coder.biases.normal_(0, 0.5)
    net.eval()
    B = 2
    torch.manual_seed(seed + 1)
    batch = torch.randn(B, C, H, W, D)
    if zero_slab:
        batch[:, :, :, :, :2] = 0                       # depth slices 0-1 are empty: masked tokens
    BD = B * D2
    feats = [torch.zeros(1).expand(BD, DIMS[0], H, W)] + \
        [torch.randn(BD, DIMS[i], H >> i, W >> i, requires_grad=True) for i in range(1, 5)]
    bb.feats = feats
    K = args.num_classes
    G = torch.randn(B, K, H, W, D)
    orig_fwd = net.voxel_fusion.forward
    net.voxel_fusion.forward = lambda vfeat, pos, mask: orig_fwd(vfeat, pos, mask, torch.Size((H2, W2, D3)))
    with R.quiet(), R.cuda_literal_to_cpu():
        y = net(batch)
    del net.voxel_fusion.forward
    gp, gi = _grads(net, (y * G).sum(), feats[1:])
    sd = {k: v.clone() for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    fx = dict(kind="seg25d", args=vars(args), bb_feat_dims=DIMS, batch=batch, feats=[f.detach() for f in feats], G=G,
              out=y.detach(), state_dict=sd, grad_params=gp, grad_feats=[None] + gi, train=False,
              stem_change=getattr(bb, "in_channels_changed", None), grid=(H2, W2, D3))
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "out", tuple(y.shape), "max|out|", float(y.abs().max()))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(4)
    gen("seg25d_stemconv", 61, _args(backbone_type="eff-tiny", orig_in_channels=4, inchan_to3_scheme="stemconv",
                                     out_fpn_upsampleD_scheme="interpolate"), C=4, D=8, zero_slab=True)
    gen("seg25d_updconv", 62, _args(backbone_type="resnet-tiny", orig_in_channels=2, inchan_to3_scheme="bridgeconv",
                                    out_fpn_upsampleD_scheme="conv", num_classes=3), C=2, D=8)
    gen("seg25d_dgroup2", 63, _args(backbone_type="resnet-tiny", orig_in_channels=1, D_groupsize=2,
                                    inchan_to3_scheme="bridgeconv", out_fpn_upsampleD_scheme="interp"), C=1, D=16)
    gen("seg25d_direct34", 64, _args(backbone_type="resnet-tiny", orig_in_channels=1, inchan_to3_scheme="bridgeconv",
                                     out_fpn_layers="34", out_fpn_upsampleD_scheme="conv", num_classes=3), C=1, D=8)
    gen("seg25d_posbias", 65, _args(backbone_type="resnet-tiny", orig_in_channels=1, inchan_to3_scheme="bridgeconv",
                                    use_squeezed_transformer=False, pos_code_type="bias", pos_bias_radius=2,
                                    out_fpn_upsampleD_scheme="conv"), C=1, D=8)


if __name__ == "__main__":
    main()
