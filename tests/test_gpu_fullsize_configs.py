"""Parity of the Squeeze-and-Expansion stack at the FULL token counts and layer widths of all five BASELINE.json configs
(SURVEY.md §8a: N = 1296 / 5184 / 1936 / 2744 / 5832), one sample each, forward AND gradients against the fp32 CPU oracle
(reference formulation).  Tolerance = BASELINE.json's north star: max|a-b| / max|b| < 1e-3 on the forward output in the
DEFAULT precision (TF32 tensor cores + the per-call-site precision policy); gradients are held to 3e-3 (they pass through
roughly twice as many TF32 contractions as the output; the 3-pass validation mode pins them to 1e-5 on the goldens).
The CPU oracle needs 10-60 s per config on the GPU box's host cores."""
import os

import pytest
import torch

from oracle import segtran_oracle as O
from tests.helpers import encoder_config, rel_err, rms_rel

pytestmark = pytest.mark.gpu

# (dims, attractors, grid, qk_bias) of BASELINE.json configs 1-5
STACKS = {
    1: ([1792, 1792], 256, (36, 36), True),
    2: ([1792, 1792, 896, 448], 256, (72, 72), False),
    3: ([2048, 2048, 2048], 256, (44, 44), True),
    4: ([1024, 1024], 1024, (14, 14, 14), True),
    5: ([1024, 1024, 1024], 2048, (18, 18, 18), True),
}


def _build(dims, A, grid, qkb, seed):
    import segtran_b200.networks.segtran_shared as S
    cfg = encoder_config(S.SegtranConfig, dims=dims, num_modes=4, num_attractors=A, pos_dim=len(grid), qk_have_bias=qkb)
    cfg.translayer_compress_ratios = [1] * len(dims)
    torch.manual_seed(seed)
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.init_weights)
    enc.apply(init.tie_qk)
    enc.apply(init.add_identity_bias)
    return enc


@pytest.mark.parametrize("cfg", [1, 2, 3, 4, 5])
def test_full_size_stack_forward_and_gradients_match_oracle(cfg):
    dims, A, grid, qkb = STACKS[cfg]
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    enc = _build(dims, A, grid, qkb, seed=20 + cfg).eval()
    p = {"voxel_fusion." + k: v.clone().requires_grad_() for k, v in enc.state_dict().items() if ".key." not in k}
    N = 1
    for s in grid:
        N *= s
    torch.manual_seed(cfg)
    x = (torch.randn(1, N, dims[0]) * 1.5 + 0.2)
    pos = O.voxels_pos_for_grid(grid, (8,) * len(grid), 1)
    mask = (torch.rand(1, N, 1) > 0.05).float() if len(grid) == 2 else torch.ones(1, N, 1)     # 2-D: zero-padded tokens
    G = torch.randn(1, N, dims[-1])
    xr = x.clone().requires_grad_()
    ref = O.fusion_encoder(p, "voxel_fusion.", xr, pos, mask, dims, 4)
    (ref * G).sum().backward()
    enc = enc.cuda()
    xg = x.cuda().requires_grad_()
    y = enc(xg, pos.cuda(), mask.cuda(), torch.Size(grid))
    (y * G.cuda()).sum().backward()
    e, r = rel_err(y, ref), rms_rel(y, ref)
    ex = rel_err(xg.grad, xr.grad)
    print("cfg%d N=%d dims=%s: fwd max-rel %.2e rms-rel %.2e | dx max-rel %.2e" % (cfg, N, dims, e, r, ex))
    assert e < 1e-3, "forward deviates from the oracle: %.3e" % e
    assert ex < 3e-3, "input gradient deviates from the oracle: %.3e" % ex
    # parameter gradients: 5e-3 of the parameter's own gradient scale plus 1e-6 of the largest gradient scale in the model (the
    # same criterion as the golden-fixture tests).  The absolute term matters for gradients that are differences of large
    # cancelling terms — the bias of the mode-softmax score (exactly zero in exact arithmetic) and the tied squeeze-out
    # Q/K weight are 1e-4 .. 1e-3 in magnitude next to 1e2 .. 1e3 for the others; on exactly these two the fp32-grade 3-pass
    # mode deviates from the fp32 CPU oracle by the same 2 .. 100 % as the default mode, i.e.
    # the fp32 reference value itself is rounding noise at that scale.
    got = dict(enc.named_parameters())
    gscale = max(float(v.grad.abs().max()) for v in p.values() if v.grad is not None)
    worst = 0.0
    for k, v in p.items():
        name = k[len("voxel_fusion."):]
        if v.grad is None or name not in got or got[name].grad is None or float(v.grad.abs().max()) == 0.0:
            continue
        gm = float(v.grad.abs().max())
        err = float((got[name].grad.cpu() - v.grad).abs().max())
        if gm > 1e-4 * gscale:
            worst = max(worst, err / gm)
        assert err <= 5e-3 * gm + 1e-6 * gscale, (name, err, gm, gscale)
    print("cfg%d: worst parameter-gradient max-rel %.2e (parameters above 1e-4 of the largest gradient scale)" % (cfg, worst))
    # no row of the fused attention was in the lower-clamp corner (csrc/sx_attn.cu)
    for layer in enc.translayers:
        assert layer.ator_out_trans.lower_clamp_ambiguous_rows == 0


@pytest.mark.parametrize("cfg", [4, 5])
def test_full_size_stack_bf16_mode_error_budget(cfg):
    """The fast bf16-operand mode (BASELINE.json config 5's precision) is NOT a parity mode: its measured deviation from the
    fp32 oracle is recorded here and bounded by its documented budget (DESIGN §2)."""
    from segtran_b200 import ops
    dims, A, grid, qkb = STACKS[cfg]
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    enc = _build(dims, A, grid, qkb, seed=40 + cfg).eval()
    p = {"voxel_fusion." + k: v.clone() for k, v in enc.state_dict().items()}
    N = 1
    for s in grid:
        N *= s
    x = torch.randn(1, N, dims[0])
    pos = O.voxels_pos_for_grid(grid, (8,) * len(grid), 1)
    mask = torch.ones(1, N, 1)
    with torch.no_grad():
        ref = O.fusion_encoder(p, "voxel_fusion.", x, pos, mask, dims, 4)
    enc = enc.cuda()
    ops.set_precision("bf16")
    try:
        with torch.no_grad():
            y = enc(x.cuda(), pos.cuda(), mask.cuda(), torch.Size(grid))
    finally:
        ops.set_precision("tf32")
    e, r = rel_err(y, ref), rms_rel(y, ref)
    print("cfg%d bf16 mode: max-rel %.2e rms-rel %.2e" % (cfg, e, r))
    assert e < 2e-2
