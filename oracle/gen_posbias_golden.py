"""Generate the tests/golden/pos*.pt fixtures of the positional-code ablations by running the REAL reference.

TEST INFRASTRUCTURE ONLY.  Run in the build container:  python -m oracle.gen_posbias_golden
Writes only the four files below; the other fixtures are left untouched.  Each holds the reference module's
state_dict, seeded inputs, the eval-mode output, the gradients of loss = (out * G).sum(), and the digests of the
seeded initial state_dict (before the zero-initialised `biases` are replaced by a seeded random table, so that the
forward exercises them).  max_pos_size is set to the grid, which keeps the reference's index buffers small; only
posbias2d.pt keeps them in its state_dict (the strict-load test), the others drop the all_* entries.
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


def gen(name, *, pos, dims, M, pd, grid, B, seed, R_=2, posw=1.0, squeeze=False, A=16, wscale=1.0, keep_index=False):
    ns = R.load()
    cfg = R.encoder_config(ns.shared, dims=dims, num_modes=M, num_attractors=A, pos_dim=pd, qk_have_bias=True)
    cfg.use_squeezed_transformer = squeeze
    cfg.pos_code_type = pos
    cfg.pos_bias_radius = R_
    cfg.pos_code_weight = posw
    cfg.max_pos_size = tuple(grid)
    enc = R.build_encoder(cfg, seed=seed).eval()
    init_digests = {k: _digest(v) for k, v in enc.state_dict().items()}
    torch.manual_seed(seed + 50)
    with torch.no_grad():
        if pos == "bias":
            b = enc.pos_code_layer.pos_coder.biases
            b.copy_(torch.randn(b.shape) * 0.5)
        if wscale != 1.0:                   # push the scores past attn_clip=500: clamp first, then the bias
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
    gp, gi = _grads(enc, (y * G).sum(), [x])
    layers = list(enc.translayers)
    max_attn = [float(t.ator_out_trans.max_attn) for t in layers] if squeeze else [float(t.max_attn) for t in layers]
    sd = {k: v.clone() for k, v in enc.state_dict().items() if keep_index or ".all_" not in k}
    fx = dict(kind="encoder_pos", pos_code_type=pos, dims=list(dims), num_modes=M, num_attractors=A, pos_dim=pd,
              qk_have_bias=True, grid=list(grid), pos_bias_radius=R_, pos_code_weight=posw,
              use_squeezed_transformer=squeeze, seed=seed, x=x.detach(), voxels_pos=vpos, vmask=mask, G=G,
              out=y.detach(), state_dict=sd, grad_params=gp, grad_x=gi[0], max_attn=max_attn,
              init_digests=init_digests)
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "N", N, "max|out|", float(y.abs().max()), "max_attn", max_attn,
          "KB", os.path.getsize(os.path.join(OUT, name + ".pt")) // 1024)


def main():
    gen("posbias3d", pos="bias", dims=[32, 32], M=4, pd=3, grid=(5, 6, 7), B=2, seed=41)
    gen("posbias2d", pos="bias", dims=[32, 32, 32], M=4, pd=2, grid=(6, 7), B=1, seed=42, posw=0.5, keep_index=True)
    gen("posbias_clamp", pos="bias", dims=[32, 32], M=4, pd=3, grid=(4, 5, 6), B=2, seed=43, wscale=40.0)
    gen("posnone_sq", pos="none", dims=[32, 32], M=4, pd=3, grid=(3, 4, 5), B=2, seed=44, squeeze=True)


if __name__ == "__main__":
    main()
