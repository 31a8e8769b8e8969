"""Generate the tests/golden/consist*.pt fixtures of the attention-consistency losses from the REAL reference.

TEST INFRASTRUCTURE ONLY.  Run in the build container:  python -m oracle.gen_consist_golden
The reference's training drivers cannot be imported (they parse arguments and import missing packages at module level),
so `attn_consist_loss_fun` is taken out of train3d.py and train2d.py with `ast` and executed on its own.  Each fixture
holds seeded score entries (the shapes SegtranFusionEncoder keeps in layers_attn_scores), the mask, orig_feat_shape,
only_first_layer, the reference loss and its gradients with respect to every score tensor.  The consist_enc* fixtures
run the reference SegtranFusionEncoder with use_attn_consist_loss=True and the reference loss on its
layers_attn_scores; they hold the encoder's state_dict (attn_scaler included), its inputs, the loss, the gradients of
every parameter and of the input, and each layer's max_attn (consist_enc_clamp: scores above attn_clip=500).
"""
from __future__ import annotations

import ast
import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import as R                      # noqa: E402
from oracle import segtran_oracle as O                  # noqa: E402
from oracle.gen_golden import OUT, _grads               # noqa: E402


def ref_loss_fun(driver):
    path = os.path.join(R.REF_CODE, driver)
    tree = ast.parse(open(path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "attn_consist_loss_fun"][0]
    ns = {"torch": torch, "F": F}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)
    return ns["attn_consist_loss_fun"]


def gen(name, *, three_d, grid, B, K, layers, A=None, only_first_layer=None, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    N = 1
    for s in grid:
        N *= s
    entries = []
    for _ in range(layers):
        if A is None:
            entries.append((torch.randn(B, 1, N, N, generator=g) * scale).requires_grad_())
        else:
            entries.append([(torch.randn(B, 1, A, N, generator=g) * scale).requires_grad_(),
                            (torch.randn(B, 1, N, A, generator=g) * scale).requires_grad_()])
    # n-hot masks at twice the token resolution (soft values after the resize)
    if three_d:
        D, H, W = grid
        lab = torch.randint(0, K, (B, 2 * H, 2 * W, 2 * D), generator=g)
        mask = F.one_hot(lab, K).permute(0, 4, 1, 2, 3).float()          # [B,K,H,W,D]
    else:
        H, W = grid
        lab = torch.randint(0, K, (B, 2 * H, 2 * W), generator=g)
        mask = F.one_hot(lab, K).permute(0, 3, 1, 2).float()
    fun = ref_loss_fun("train3d.py" if three_d else "train2d.py")
    kw = {} if only_first_layer is None else {"only_first_layer": only_first_layer}
    loss = fun(entries, torch.Size(grid), mask, **kw)
    loss.backward()
    flat = [t for e in entries for t in (e if isinstance(e, list) else [e])]
    fx = {"three_d": three_d, "grid": tuple(grid), "mask": mask,
          "entries": [[t.detach() for t in e] if isinstance(e, list) else e.detach() for e in entries],
          "only_first_layer": only_first_layer, "loss": loss.detach(),
          "grads": [torch.zeros_like(t) if t.grad is None else t.grad for t in flat]}
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, float(loss))


def _seg_mask(g, B, K, grid, three_d):
    """n-hot mask at twice the token resolution: [B,K,H,W,D] (3-D, grid = (D2,H2,W2)) or [B,K,H,W]."""
    if three_d:
        D, H, W = grid
        lab = torch.randint(0, K, (B, 2 * H, 2 * W, 2 * D), generator=g)
        return F.one_hot(lab, K).permute(0, 4, 1, 2, 3).float()
    H, W = grid
    lab = torch.randint(0, K, (B, 2 * H, 2 * W), generator=g)
    return F.one_hot(lab, K).permute(0, 3, 1, 2).float()


def gen_encoder(name, *, three_d, dims, grid, B, K, seed, squeeze=True, M=4, A=16, only_first_layer=None, wscale=1.0,
                scaler_scale=1.0):
    ns = R.load()
    pd = len(grid)
    cfg = R.encoder_config(ns.shared, dims=dims, num_modes=M, num_attractors=A, pos_dim=pd, qk_have_bias=True)
    cfg.use_squeezed_transformer = squeeze
    cfg.use_attn_consist_loss = True
    enc = R.build_encoder(cfg, seed=seed).eval()
    with torch.no_grad():
        for n, p in enc.named_parameters():
            if wscale != 1.0 and n.endswith("query.weight"):       # scores past attn_clip = 500: the clamp fires
                p.mul_(wscale)
            if scaler_scale != 1.0 and n.startswith("attn_scaler") and n.endswith("weight"):
                p.mul_(scaler_scale)
    N = 1
    for s_ in grid:
        N *= s_
    g = torch.Generator().manual_seed(seed + 100)
    x = torch.randn(B, N, dims[0], generator=g, requires_grad=True)
    vpos = O.voxels_pos_for_grid(grid, (8,) * pd, B)
    vmask = (torch.rand(B, N, 1, generator=g) > 0.2).long()
    mask = _seg_mask(g, B, K, grid, three_d)
    with R.quiet():
        enc(x, vpos, vmask, torch.Size(grid))
    fun = ref_loss_fun("train3d.py" if three_d else "train2d.py")
    kw = {} if only_first_layer is None else {"only_first_layer": only_first_layer}
    loss = fun(enc.layers_attn_scores, torch.Size(grid), mask, **kw)
    gp, gi = _grads(enc, loss, [x])
    layers = list(enc.translayers)
    mods = [m for t in layers for m in ((t.in_ator_trans, t.ator_out_trans) if squeeze else (t,))]
    fx = dict(kind="consist_encoder", three_d=three_d, dims=list(dims), num_modes=M, num_attractors=A, pos_dim=pd,
              qk_have_bias=True, use_squeezed_transformer=squeeze, grid=tuple(grid), only_first_layer=only_first_layer,
              x=x.detach(), voxels_pos=vpos, vmask=vmask, mask=mask, state_dict={k: v.clone() for k, v in
                                                                                  enc.state_dict().items()},
              loss=loss.detach(), grad_params=gp, grad_x=gi[0], max_attn=[float(m.max_attn) for m in mods])
    torch.save(fx, os.path.join(OUT, name + ".pt"))
    print(name, "loss", float(loss), "max_attn", [round(v, 1) for v in fx["max_attn"]])


def main():
    gen("consist3d_pair", three_d=True, grid=(5, 6, 7), B=2, K=3, layers=1, A=37, scale=0.3, seed=1)
    gen("consist3d_pair2", three_d=True, grid=(4, 6, 6), B=2, K=2, layers=2, A=24, only_first_layer=False, scale=0.3,
        seed=2)
    gen("consist2d_pair", three_d=False, grid=(12, 14), B=2, K=3, layers=2, A=20, scale=0.05, seed=3)
    gen("consist2d_pair_cap", three_d=False, grid=(12, 14), B=2, K=3, layers=2, A=20, scale=1.0, seed=4)
    gen("consist2d_dense", three_d=False, grid=(10, 13), B=2, K=4, layers=2, scale=1.0, seed=5)
    gen("consist3d_dense", three_d=True, grid=(4, 5, 6), B=2, K=2, layers=2, only_first_layer=False, scale=2.0, seed=6)
    gen_encoder("consist_enc3d", three_d=True, dims=[32, 32], grid=(5, 6, 7), B=2, K=3, seed=61)
    gen_encoder("consist_enc3d_2l", three_d=True, dims=[32, 32, 32], grid=(4, 5, 6), B=2, K=2, seed=62,
                only_first_layer=False)
    gen_encoder("consist_enc2d", three_d=False, dims=[32, 32, 32], grid=(12, 14), B=2, K=3, seed=63,
                scaler_scale=0.02)
    gen_encoder("consist_enc2d_cap", three_d=False, dims=[32, 32, 32], grid=(12, 14), B=2, K=3, seed=64,
                scaler_scale=200.0)
    gen_encoder("consist_enc2d_dense", three_d=False, dims=[32, 32], grid=(10, 13), B=2, K=4, seed=65, squeeze=False)
    gen_encoder("consist_enc3d_dense", three_d=True, dims=[32, 32, 32], grid=(4, 5, 6), B=2, K=2, seed=66,
                squeeze=False, only_first_layer=False)
    gen_encoder("consist_enc_clamp", three_d=True, dims=[32, 32], grid=(4, 5, 6), B=2, K=3, seed=67, wscale=40.0)


if __name__ == "__main__":
    main()
