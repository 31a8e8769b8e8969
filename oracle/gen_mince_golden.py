"""Generate the tests/golden/mince*.pt fixtures of the mince transformer (--mince --nosqueeze) by running the REAL reference.

TEST INFRASTRUCTURE ONLY.  Run in the build container:  python -m oracle.gen_mince_golden
Writes only the five files below; the other fixtures are left untouched.  Each holds the reference module's state_dict,
seeded inputs, the eval-mode output, the gradients of loss = (out * G).sum(), the per-layer, per-scale max_attn /
clamp_count, and the digests of the seeded initial state_dict (taken before the zero-initialised per-scale `biases` are
replaced by seeded random tables, so that the forward exercises them).  max_pos_size is set to the full grid; only
mince2d.pt keeps the reference's index buffers in its state_dict (the strict-load test).
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import as R                      # noqa: E402
from oracle import segtran_oracle as O                  # noqa: E402
from oracle.gen_golden import OUT, _digest, _grads     # noqa: E402


def gen(name, *, pos, dims, M, pd, grid, B, seed, scales, props, R_=2, posw=1.0, qscale=1.0, keep_index=False):
    ns = R.load()
    cfg = R.encoder_config(ns.shared, dims=dims, num_modes=M, num_attractors=16, pos_dim=pd, qk_have_bias=True)
    cfg.use_squeezed_transformer = False
    cfg.use_mince_transformer = True
    cfg.mince_scales = list(scales)
    cfg.mince_channel_props = list(props)
    cfg.pos_code_type = pos
    cfg.pos_bias_radius = R_
    cfg.pos_code_weight = posw
    cfg.max_pos_size = tuple(grid)
    enc = R.build_encoder(cfg, seed=seed).eval()
    init_digests = {k: _digest(v) for k, v in enc.state_dict().items()}
    torch.manual_seed(seed + 50)
    with torch.no_grad():
        if pos == "bias":
            for layer in enc.pos_code_layers:
                b = layer.pos_coder.biases
                b.copy_(torch.randn(b.shape) * 0.5)
        if qscale != 1.0:                   # push the first scale's scores past attn_clip=500, not the others'
            for t in enc.translayers:
                d = t.attention_mode_dim
                hi = t.mince_qk_channel_indices[1]
                for m in range(M):
                    t.query.weight[m * d:m * d + hi].mul_(qscale)
                    t.key.weight[m * d:m * d + hi].mul_(qscale)
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
    gp, gi = _grads(enc, (y * G).sum(), [x])
    layers = list(enc.translayers)
    max_attn = [[float(v) for v in t.max_attn] for t in layers]
    clamp_count = [[int(v) for v in t.clamp_count] for t in layers]
    sd = {k: v.clone() for k, v in enc.state_dict().items() if keep_index or ".all_" not in k}
    fx = dict(kind="encoder_mince", pos_code_type=pos, dims=list(dims), num_modes=M, num_attractors=16, pos_dim=pd,
              qk_have_bias=True, grid=list(grid), pos_bias_radius=R_, pos_code_weight=posw, mince_scales=list(scales),
              mince_channel_props=list(props), use_squeezed_transformer=False, seed=seed, x=x.detach(),
              voxels_pos=vpos, vmask=mask, G=G, out=y.detach(), state_dict=sd, grad_params=gp, grad_x=gi[0],
              max_attn=max_attn, clamp_count=clamp_count, init_digests=init_digests)
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "N", N, "max|out|", float(y.abs().max()), "max_attn", max_attn, "clamp", clamp_count,
          "KB", os.path.getsize(os.path.join(OUT, name + ".pt")) // 1024)


def main():
    gen("mince3d", pos="bias", dims=[32, 32], M=4, pd=3, grid=(5, 6, 7), B=2, seed=61, scales=[1, 2], props=[3, 1])
    gen("mince2d", pos="bias", dims=[32, 32, 32], M=4, pd=2, grid=(8, 9), B=1, seed=62, scales=[4, 2, 1],
        props=[1, 1, 2], R_=1, posw=0.5, keep_index=True)
    gen("mince_lsinu", pos="lsinu", dims=[32, 32], M=4, pd=3, grid=(6, 6, 8), B=1, seed=63, scales=[1, 2, 3],
        props=[1, 1, 1])
    gen("mince_none", pos="none", dims=[32, 32], M=4, pd=2, grid=(9, 10), B=2, seed=64, scales=[1, 3], props=[1, 1])
    gen("mince_clamp", pos="bias", dims=[32, 32], M=4, pd=3, grid=(4, 5, 6), B=2, seed=65, scales=[1, 2],
        props=[1, 1], qscale=150.0)


if __name__ == "__main__":
    main()
