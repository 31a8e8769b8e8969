"""Generate the tests/golden/seg*_direct* fixtures of the class head without the out-FPN (out_fpn_layers ==
in_fpn_layers) from the REAL reference shells.

TEST INFRASTRUCTURE ONLY.  Run in the build container:  python -m oracle.gen_direct_head_golden
Same recipe as gen_head_golden (fixed-feature backbones, loss = (out * G).sum(), feature widths [8, 8, 16, 16, 32],
2 modes), 3 classes so the head has 12 sub-pixel rows.  The input batch only sets the shapes and the nonzero mask, so
it is stored as an expanded tensor of ones, and the unused level-0 feature map as expanded zeros.  Fixtures:
  seg2d_direct34          --infpn 34 --outfpn 34, 32x32 images, eval mode
  seg2d_direct234         --infpn 234 --outfpn 234 (the transposed conv on the 1/4-resolution grid), eval mode
  seg3d_direct34          --infpn 34 --outfpn 34, (H,W,D) = (16,16,24) volumes, D_pool_K = 2: token grid
                          (D2,H2,W2) = (3,2,2), eval mode
  seg3d_direct34_outdrop  the same with --outdrop, train mode, dropout 0 (the option has no map to act on)
Each fixture holds the digests of the shell's non-backbone parameters as built from the seed (and, in 3-D, the torch
RNG states right after the reference's I3D backbone is constructed and after init_weights has visited it).
"""
from __future__ import annotations

import os
import sys
from argparse import Namespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import as R                                                # noqa: E402
from oracle.gen_golden import OUT, FixedFeatBackbone2d, FixedFeatBackbone3d, _digest, _grads   # noqa: E402

DIMS = [8, 8, 16, 16, 32]
K = 3


def gen_seg3d(name, outdrop, seed):
    ns = R.load()
    import networks.aj_i3d.aj_i3d as aj
    ns.shared.bb2feat_dims["i3d-tiny"] = DIMS
    args = Namespace(num_classes=K, backbone_type="i3d-tiny", use_pretrained=False, num_attractors=12,
                     num_translayers=1, num_modes=2, trans_output_type="private", mid_type="shared",
                     orig_in_channels=4, D_pool_K=2, inchan_to3_scheme="bridgeconv", D_groupsize=1, device="cpu",
                     in_fpn_layers="34", out_fpn_layers="34", in_fpn_scheme="AN", out_fpn_scheme="AN",
                     translayer_compress_ratios=[1, 1], dropout_prob=0.0, tie_qk_scheme="shared",
                     qk_have_bias=True, use_squeezed_transformer=True, pos_code_type="lsinu",
                     out_fpn_upsampleD_scheme="interp", out_fpn_do_dropout=outdrop)
    states = {}
    orig_init, orig_apply = aj.InceptionI3d.__init__, aj.InceptionI3d.apply

    def init(self, *a, **k):
        orig_init(self, *a, **k)
        states.setdefault("built", torch.get_rng_state())

    def apply(self, fn):
        out = orig_apply(self, fn)
        states.setdefault("applied", torch.get_rng_state())
        return out

    aj.InceptionI3d.__init__, aj.InceptionI3d.apply = init, apply
    try:
        torch.manual_seed(seed)
        with R.quiet():
            ns.seg3d.CONFIG.update_config(args)
            net = ns.seg3d.Segtran3d(ns.seg3d.CONFIG)
    finally:
        aj.InceptionI3d.__init__, aj.InceptionI3d.apply = orig_init, orig_apply
    assert not net.do_out_fpn and isinstance(net.out_conv3d, torch.nn.ConvTranspose3d)
    sd0 = net.state_dict()
    init_digests = {k: _digest(v) for k, v in sd0.items() if not k.startswith("backbone.")}
    net.train() if outdrop else net.eval()
    B, (H, W, D) = 2, (16, 16, 24)
    c = ns.shared.bb2feat_dims["i3d-tiny"]
    torch.manual_seed(seed + 1)
    batch = torch.ones(1).expand(B, 4, H, W, D)
    # (D, H, W) feature maps of the frames-first backbone; levels 1-2 feed only the out-FPN, which this head skips
    feats = [torch.zeros(1).expand(B, c[0], 12, 8, 8), torch.randn(B, c[1], 12, 8, 8), torch.randn(B, c[2], 12, 4, 4),
             torch.randn(B, c[3], 6, 2, 2), torch.randn(B, c[4], 3, 1, 1)]
    feats = feats[:1] + [f.requires_grad_(True) for f in feats[1:]]
    net.backbone = FixedFeatBackbone3d(feats)
    G = torch.randn(B, K, H, W, D)
    with R.quiet(), R.cuda_literal_to_cpu():
        y = net(batch)
    gp, gi = _grads(net, (y * G).sum(), feats[1:])
    sd = {k: v.clone() for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    fx = dict(kind="seg3d", args=vars(args), bb_feat_dims=c, batch=batch, feats=[f.detach() for f in feats], G=G,
              out=y.detach(), state_dict=sd, grad_params=gp, grad_feats=[None] + gi, train=bool(outdrop),
              init_seed=seed, init_digests=init_digests, rng_built=states["built"], rng_applied=states["applied"])
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "out", tuple(y.shape), "max|out|", float(y.abs().max()))


def gen_seg2d(name, layers, seed):
    ns = R.load()
    ns.shared.bb2feat_dims["resnet-tiny"] = DIMS
    args = Namespace(num_classes=K, backbone_type="resnet-tiny", use_pretrained=False, num_attractors=10,
                     num_translayers=1, num_modes=2, trans_output_type="private", mid_type="shared",
                     device="cpu", in_fpn_layers=layers, out_fpn_layers=layers, in_fpn_scheme="AN",
                     out_fpn_scheme="AN", translayer_compress_ratios=[1, 1], dropout_prob=0.0,
                     tie_qk_scheme="shared", qk_have_bias=False, use_squeezed_transformer=True,
                     pos_code_type="lsinu", use_global_bias=False, num_modalities=0, out_fpn_do_dropout=False)
    import resnet as ref_resnet
    ref_resnet.__dict__["resnet-tiny"] = lambda pretrained=False, do_pool1=True: torch.nn.Identity()
    torch.manual_seed(seed)
    with R.quiet():
        ns.seg2d.CONFIG.update_config(args)
        net = ns.seg2d.Segtran2d(ns.seg2d.CONFIG)
    assert not net.do_out_fpn and isinstance(net.out_conv, torch.nn.ConvTranspose2d)
    init_digests = {k: _digest(v) for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    net.eval()
    B, S = 2, 32
    c = ns.shared.bb2feat_dims["resnet-tiny"]
    torch.manual_seed(seed + 1)
    batch = torch.ones(1).expand(B, 3, S, S)
    feats = [torch.zeros(1).expand(B, c[0], 16, 16), torch.randn(B, c[1], 16, 16), torch.randn(B, c[2], 8, 8),
             torch.randn(B, c[3], 4, 4), torch.randn(B, c[4], 2, 2)]
    feats = feats[:1] + [f.requires_grad_(True) for f in feats[1:]]
    net.backbone = FixedFeatBackbone2d(feats)
    G = torch.randn(B, K, S, S)
    with R.quiet():
        y = net(batch)
    gp, gi = _grads(net, (y * G).sum(), feats[1:])
    sd = {k: v.clone() for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    fx = dict(kind="seg2d", args=vars(args), bb_feat_dims=c, batch=batch, feats=[f.detach() for f in feats], G=G,
              out=y.detach(), state_dict=sd, grad_params=gp, grad_feats=[None] + gi, train=False,
              init_seed=seed, init_digests=init_digests)
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "out", tuple(y.shape), "max|out|", float(y.abs().max()))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(4)
    gen_seg2d("seg2d_direct34", "34", seed=51)
    gen_seg2d("seg2d_direct234", "234", seed=52)
    gen_seg3d("seg3d_direct34", False, seed=53)
    gen_seg3d("seg3d_direct34_outdrop", True, seed=54)


if __name__ == "__main__":
    main()
