"""Generate the tests/golden/seg25d_outdrop_*.pt fixtures of the 2.5-D --outdrop head from the REAL reference Segtran25d.

TEST INFRASTRUCTURE ONLY.  Run in the build container:  python -m oracle.gen_seg25d_outdrop_golden
Same stand-in backbones, patches, sizes and loss as oracle/gen_seg25d_golden.py (whose fixtures this leaves alone), but
the reference shell runs in train mode with out_fpn_do_dropout=True and dropout 0, as oracle/gen_head_golden.py does
for the 3-D model: the out-FPN dropout is then the identity and the fixture pins everything around it.  Cases:
  seg25d_outdrop_updconv   --upd conv, 3 classes (the interleaved depth unfold)
  seg25d_outdrop_interp    --upd interpolate (linear x D_pool_K)
  seg25d_outdrop_noupd     --upd interp (the drivers' default, no depth map in the reference)
  seg25d_outdrop_dk1       --upd conv with D_pool_K = 1 (no depth map either)
  seg25d_outdrop_k5        --upd conv, 5 classes (more than one class chunk of the dropout head)
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import as R                                                # noqa: E402
from oracle.gen_golden import OUT, _grads                                        # noqa: E402
from oracle.gen_seg25d_golden import DIMS, H, W, FixedFeatEff, FixedFeatRes, _args   # noqa: E402


def gen(name, seed, args, C, D):
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
    D2 = D // args.D_groupsize
    H2, W2, D3 = H // 8, W // 8, D2 // args.D_pool_K
    cfg.pos_code_every_layer = True
    cfg.max_pos_size = (H2, W2, D3)
    torch.manual_seed(seed)
    try:
        with R.quiet():
            cfg.update_config(args)
            net = seg25d.Segtran25d(cfg)
    finally:
        seg25d.EfficientNet.from_name = orig_from_name
    assert net.out_fpn_do_dropout and net.out_fpn_dropout.p == 0.0
    bb = net.backbone
    net.train()
    B = 2
    torch.manual_seed(seed + 1)
    batch = torch.randn(B, C, H, W, D)
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
              out=y.detach(), state_dict=sd, grad_params=gp, grad_feats=[None] + gi, train=True,
              stem_change=getattr(bb, "in_channels_changed", None), grid=(H2, W2, D3))
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "out", tuple(y.shape), "max|out|", float(y.abs().max()))


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(4)
    common = dict(backbone_type="resnet-tiny", orig_in_channels=2, inchan_to3_scheme="bridgeconv",
                  out_fpn_do_dropout=True)
    gen("seg25d_outdrop_updconv", 71, _args(out_fpn_upsampleD_scheme="conv", num_classes=3, **common), C=2, D=8)
    gen("seg25d_outdrop_interp", 72, _args(out_fpn_upsampleD_scheme="interpolate", **common), C=2, D=8)
    gen("seg25d_outdrop_noupd", 73, _args(out_fpn_upsampleD_scheme="interp", **common), C=2, D=8)
    gen("seg25d_outdrop_dk1", 74, _args(out_fpn_upsampleD_scheme="conv", D_pool_K=1, **common), C=2, D=4)
    gen("seg25d_outdrop_k5", 75, _args(out_fpn_upsampleD_scheme="conv", num_classes=5, **common), C=2, D=8)


if __name__ == "__main__":
    main()
