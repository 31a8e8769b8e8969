"""Generate the tests/golden/multihead_*.pt fixtures of the multi-head ablation (--nosqueeze --multihead) by running the
REAL reference.

TEST INFRASTRUCTURE ONLY.  Run in the build container:  python -m oracle.gen_multihead_golden
Writes only the files below; the other fixtures are left untouched.  Each encoder fixture holds the reference module's
state_dict, seeded inputs, the eval-mode output, the gradients of loss = (out * G).sum() (of the reference's attention-
consistency loss for multihead_consist), every layer's max_attn, and the digests of the seeded initial state_dict (taken
before a positional-bias table is replaced by a seeded random one).  The shell fixtures run the reference Segtran2d /
Segtran3d with --nosqueeze --multihead on the fixed-feature backbones of seg2d_tiny / seg3d_tiny, whose inputs (batch,
backbone features, G) they use and do not repeat; they keep the logits and the feature gradients as the values at a seeded
sample of elements, with each tensor's max|.| (see _sampled), which keeps the files small.
"""
from __future__ import annotations

import os
import sys
from argparse import Namespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import as R                      # noqa: E402
from oracle import segtran_oracle as O                  # noqa: E402
from oracle.gen_consist_golden import _seg_mask, ref_loss_fun     # noqa: E402
from oracle.gen_golden import OUT, FixedFeatBackbone2d, FixedFeatBackbone3d, _digest, _grads     # noqa: E402


def gen(name, *, dims, grid, B, seed, M=4, qkb=True, pos="lsinu", out_type="private", R_=2, posw=1.0, wscale=1.0,
        consist=False, K=3):
    ns = R.load()
    pd = len(grid)
    cfg = R.encoder_config(ns.shared, dims=dims, num_modes=M, num_attractors=16, pos_dim=pd, qk_have_bias=qkb,
                           trans_output_type=out_type)
    cfg.use_squeezed_transformer = False                 # what the drivers do with --multihead (train2d.py:259-260)
    cfg.ablate_multihead = True
    cfg.pos_code_type = pos
    cfg.pos_bias_radius = R_
    cfg.pos_code_weight = posw
    cfg.max_pos_size = tuple(grid)
    cfg.use_attn_consist_loss = consist
    enc = R.build_encoder(cfg, seed=seed).eval()
    init_digests = {k: _digest(v) for k, v in enc.state_dict().items()}
    layer_num_modes = [t.config.num_modes for t in enc.translayers]
    torch.manual_seed(seed + 50)
    with torch.no_grad():
        if pos == "bias":
            b = enc.pos_code_layer.pos_coder.biases
            b.copy_(torch.randn(b.shape) * 0.5)
        if wscale != 1.0:                   # push the scores past attn_clip=500 (segtran_shared.py:578-580)
            for n, p in enc.named_parameters():
                if n.endswith("query.weight"):
                    p.mul_(wscale)
    N = 1
    for g in grid:
        N *= g
    torch.manual_seed(seed + 100)
    x = torch.randn(B, N, dims[0], requires_grad=True)
    vpos = O.voxels_pos_for_grid(grid, (8,) * pd, B)
    mask = (torch.rand(B, N, 1) > 0.2).long()
    G = torch.randn(B, N, dims[-1])
    with R.quiet():
        y = enc(x, vpos, mask, torch.Size(grid))
    fx = dict(kind="encoder_multihead", dims=list(dims), num_modes=M, num_attractors=16, pos_dim=pd, qk_have_bias=qkb,
              grid=list(grid), pos_code_type=pos, pos_bias_radius=R_, pos_code_weight=posw, trans_output_type=out_type,
              use_attn_consist_loss=consist, seed=seed, x=x.detach(), voxels_pos=vpos, vmask=mask, out=y.detach(),
              init_digests=init_digests, layer_num_modes=layer_num_modes)
    if consist:
        three_d = pd == 3
        seg = _seg_mask(torch.Generator().manual_seed(seed + 200), B, K, grid, three_d)
        loss = ref_loss_fun("train3d.py" if three_d else "train2d.py")(enc.layers_attn_scores, torch.Size(grid), seg)
        fx.update(seg_mask=seg, three_d=three_d, loss=loss.detach())
    else:
        loss = (y * G).sum()
        fx.update(G=G)
    gp, gi = _grads(enc, loss, [x])
    fx.update(state_dict={k: v.clone() for k, v in enc.state_dict().items() if ".all_" not in k}, grad_params=gp,
              grad_x=gi[0], max_attn=[float(t.max_attn) for t in enc.translayers])
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "N", N, "max|out|", float(y.detach().abs().max()), "max_attn", fx["max_attn"],
          "KB", os.path.getsize(os.path.join(OUT, name + ".pt")) // 1024)


SAMPLES = 8192


def _sampled(t, seed=20240601):
    """A large shell tensor as the values at a fixed, seeded sample of flat indices (all of them for a small one) plus
    its max|.| over every element, so that a check of max|a-b| / max|b| on the sample uses the full tensor's scale."""
    flat = t.detach().reshape(-1)
    if flat.numel() <= 2 * SAMPLES:
        idx = torch.arange(flat.numel(), dtype=torch.int32)
    else:
        g = torch.Generator().manual_seed(seed)
        idx = torch.randperm(flat.numel(), generator=g)[:SAMPLES].sort().values.to(torch.int32)
    return dict(shape=tuple(t.shape), idx=idx, val=flat[idx.long()].clone(), absmax=float(flat.abs().max()))


def _check_inputs(name, batch, feats, G):
    """The shell fixtures draw the inputs of `name` (same seeds) and keep only a reference to them."""
    fx = torch.load(os.path.join(OUT, name + ".pt"), map_location="cpu", weights_only=False)
    assert torch.equal(fx["batch"], batch) and torch.equal(fx["G"], G)
    assert all(torch.equal(a, b.detach()) for a, b in zip(fx["feats"], feats))


def gen_seg3d(name, seed=3):
    """seg3d_tiny's shell and backbone features with --nosqueeze --multihead."""
    ns = R.load()
    ns.shared.bb2feat_dims["i3d-tiny"] = [8, 16, 24, 32, 48]
    args = Namespace(num_classes=4, backbone_type="i3d-tiny", use_pretrained=False, num_attractors=12,
                     num_translayers=1, num_modes=4, trans_output_type="private", mid_type="shared",
                     orig_in_channels=4, D_pool_K=2, inchan_to3_scheme="bridgeconv", D_groupsize=1, device="cpu",
                     in_fpn_layers="34", out_fpn_layers="1234", in_fpn_scheme="AN", out_fpn_scheme="AN",
                     translayer_compress_ratios=[1, 1], dropout_prob=0.0, tie_qk_scheme="shared",
                     qk_have_bias=True, use_squeezed_transformer=False, pos_code_type="lsinu", ablate_multihead=True)
    torch.manual_seed(seed)
    with R.quiet():
        ns.seg3d.CONFIG.update_config(args)
        net = ns.seg3d.Segtran3d(ns.seg3d.CONFIG)
    net.eval()
    B, S = 2, 32
    c = ns.shared.bb2feat_dims["i3d-tiny"]
    torch.manual_seed(seed + 1)
    batch = torch.randn(B, 4, S, S, S)
    batch[:, :, :, :, :8] = 0
    feats = [torch.randn(B, c[0], 16, 16, 16), torch.randn(B, c[1], 16, 16, 16), torch.randn(B, c[2], 16, 8, 8),
             torch.randn(B, c[3], 8, 4, 4), torch.randn(B, c[4], 4, 2, 2)]
    feats = [f.requires_grad_(True) for f in feats]
    net.backbone = FixedFeatBackbone3d(feats)
    G = torch.randn(B, 4, S, S, S)
    with R.quiet(), R.cuda_literal_to_cpu():
        y = net(batch)
    gp, gi = _grads(net, (y * G).sum(), feats[1:])
    sd = {k: v.clone() for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    _check_inputs("seg3d_tiny", batch, feats, G)
    fx = dict(kind="seg3d", args=vars(args), bb_feat_dims=c, inputs="seg3d_tiny", out=_sampled(y), state_dict=sd,
              grad_params=gp, grad_feats=[None] + [_sampled(g) for g in gi])
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "out", tuple(y.shape), "max|out|", float(y.detach().abs().max()))


def gen_seg2d(name, seed=4):
    """seg2d_tiny's shell and backbone features with --nosqueeze --multihead (two layers, the second compressed)."""
    ns = R.load()
    ns.shared.bb2feat_dims["resnet-tiny"] = [8, 16, 24, 32, 48]
    args = Namespace(num_classes=3, backbone_type="resnet-tiny", use_pretrained=False, num_attractors=10,
                     num_translayers=2, num_modes=4, trans_output_type="private", mid_type="shared",
                     device="cpu", in_fpn_layers="34", out_fpn_layers="1234", in_fpn_scheme="AN",
                     out_fpn_scheme="AN", translayer_compress_ratios=[1, 1, 2], dropout_prob=0.0,
                     tie_qk_scheme="shared", qk_have_bias=False, use_squeezed_transformer=False,
                     pos_code_type="lsinu", use_global_bias=False, num_modalities=0, ablate_multihead=True)
    import resnet as ref_resnet
    ref_resnet.__dict__["resnet-tiny"] = lambda pretrained=False, do_pool1=True: torch.nn.Identity()
    torch.manual_seed(seed)
    with R.quiet():
        ns.seg2d.CONFIG.update_config(args)
        net = ns.seg2d.Segtran2d(ns.seg2d.CONFIG)
    net.eval()
    B, S = 2, 64
    c = ns.shared.bb2feat_dims["resnet-tiny"]
    torch.manual_seed(seed + 1)
    batch = torch.randn(B, 3, S, S)
    batch[:, :, :16, :] = 0
    feats = [torch.randn(B, c[0], 32, 32), torch.randn(B, c[1], 32, 32), torch.randn(B, c[2], 16, 16),
             torch.randn(B, c[3], 8, 8), torch.randn(B, c[4], 4, 4)]
    feats = [f.requires_grad_(True) for f in feats]
    net.backbone = FixedFeatBackbone2d(feats)
    G = torch.randn(B, 3, S, S)
    with R.quiet():
        y = net(batch)
    gp, gi = _grads(net, (y * G).sum(), feats[1:])
    sd = {k: v.clone() for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    _check_inputs("seg2d_tiny", batch, feats, G)
    fx = dict(kind="seg2d", args=vars(args), bb_feat_dims=c, inputs="seg2d_tiny", out=_sampled(y), state_dict=sd,
              grad_params=gp, grad_feats=[None] + [_sampled(g) for g in gi])
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "out", tuple(y.shape), "max|out|", float(y.detach().abs().max()))


def main():
    torch.set_num_threads(4)
    gen("multihead_2d", dims=[64, 64], grid=(12, 12), B=2, seed=71)                       # N = 144 > 128 keys
    gen("multihead_3d_compress", dims=[64, 64, 32], grid=(3, 4, 5), B=2, seed=72, qkb=False)     # C != F, dh = 8
    gen("multihead_sharedout", dims=[64, 64], grid=(3, 4, 5), B=2, seed=73, out_type="shared")
    gen("multihead_posbias", dims=[32, 32], grid=(4, 5, 6), B=2, seed=74, pos="bias", posw=0.5)
    gen("multihead_posnone", dims=[32, 32], grid=(9, 10), B=2, seed=75, pos="none")
    gen("multihead_clamp", dims=[64, 64], grid=(3, 4, 5), B=1, seed=76, wscale=60.0)
    gen("multihead_consist", dims=[32, 32, 32], grid=(4, 5, 6), B=2, seed=77, consist=True)
    gen("multihead_d9", dims=[36, 36], grid=(3, 4, 5), B=2, seed=78)                     # d = dh = 9
    gen_seg3d("multihead_seg3d")
    gen_seg2d("multihead_seg2d")


if __name__ == "__main__":
    main()
