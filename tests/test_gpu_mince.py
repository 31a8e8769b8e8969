"""The mince transformer (--mince --nosqueeze) on the GPU: the token-grid resampling kernels against float64
F.interpolate and its autograd, the encoder against the reference's fixtures (oracle/gen_mince_golden.py) and against the
float64 oracle, and the training-mode properties (determinism, direct accumulation, CUDA-graph replay)."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from segtran_b200 import ops  # noqa: E402
import segtran_b200.networks.segtran_shared as S  # noqa: E402
from oracle import mince_oracle as MO  # noqa: E402
from tests.helpers import encoder_config  # noqa: E402

DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ["mince3d", "mince2d", "mince_lsinu", "mince_none", "mince_clamp"]


# ---------------------------------------------------------------------------------------------------------------------
# resampling kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid,scale", [((5, 6, 7), 2), ((6, 6, 8), 3), ((8, 9), 4), ((9, 10), 3), ((7, 5), 1)])
def test_downsample_windows_match_interpolate(grid, scale):
    torch.manual_seed(0)
    B, G, D = 2, 3, 19
    N = math.prod(grid)
    x = torch.randn(B, N, G * D, device=DEV, requires_grad=True)
    g_out = S.mince_grids(grid, [scale])[0]
    wins = [(0, 5), (5, 13), (13, 19)]                  # unaligned offsets, widths 5 / 8 / 6 -> padded to 8 / 8 / 8
    ratios = [(ops.down_ratio(scale),) * len(grid)] * 3
    ys = ops.resize_tokens(x, G, grid, [g_out] * 3, ratios, wins, round_out=False)
    dys = [torch.randn_like(y) for y in ys]
    sum((y * dy).sum() for y, dy in zip(ys, dys)).backward()
    x64 = x.detach().double().cpu().requires_grad_()
    loss = 0
    for (c0, c1), y, dy in zip(wins, ys, dys):
        w = c1 - c0
        ref = MO.resample(x64.view(B, N, G, D).permute(0, 2, 1, 3)[..., c0:c1], grid, scale)    # [B,G,Ns,w]
        ours = y.view(B, -1, G, y.shape[-1] // G).permute(0, 2, 1, 3)
        assert ours.shape[-1] == 8 and torch.all(ours[..., w:] == 0)                                   # padding is zero
        torch.testing.assert_close(ours[..., :w].double().cpu(), ref.detach(), rtol=1e-5, atol=1e-5)
        loss = loss + (ref * dy.view(B, -1, G, 8).permute(0, 2, 1, 3)[..., :w].double().cpu()).sum()
    loss.backward()
    torch.testing.assert_close(x.grad.double().cpu(), x64.grad, rtol=1e-5, atol=1e-5)
    # the adjoint is a gather in a fixed order: bit-identical across runs
    g1 = x.grad.clone()
    x.grad = None
    ys = ops.resize_tokens(x, G, grid, [g_out] * 3, ratios, wins, round_out=False)
    sum((y * dy).sum() for y, dy in zip(ys, dys)).backward()
    assert torch.equal(g1, x.grad)


@pytest.mark.parametrize("grid,scales", [((5, 6, 7), [1, 2]), ((6, 6, 8), [1, 2, 3]), ((8, 9), [4, 2, 1])])
def test_upsample_into_windows_of_a_wider_tensor(grid, scales):
    torch.manual_seed(1)
    B, G, Fd = 2, 4, 29
    grids = S.mince_grids(grid, scales)
    idx, _ = S.fracs_to_indices(Fd, [1] * len(scales))
    wins = [(idx[s], idx[s + 1]) for s in range(len(scales))]
    us = [torch.randn(B, G, math.prod(g), ops._pad4(b - a), device=DEV, requires_grad=True) for g, (a, b) in zip(grids, wins)]
    U = ops.resize_tokens_into(us, grid, grids, wins, Fd, round_out=False)
    dU = torch.randn_like(U)
    (U * dU).sum().backward()
    refs = []
    u64 = [u.detach().double().cpu().requires_grad_() for u in us]
    for u, g, (a, b) in zip(u64, grids, wins):
        refs.append(MO.resample(u[..., :b - a], g, size=grid))
    ref = torch.cat(refs, -1)
    torch.testing.assert_close(U.detach().double().cpu(), ref.detach(), rtol=1e-5, atol=1e-5)
    (ref * dU.double().cpu()).sum().backward()
    for u, r, (a, b) in zip(us, u64, wins):
        torch.testing.assert_close(u.grad[..., :b - a].double().cpu(), r.grad[..., :b - a], rtol=1e-5, atol=1e-5)
        assert torch.all(u.grad[..., b - a:] == 0)


# ---------------------------------------------------------------------------------------------------------------------
# against the fixtures made by the reference
# ---------------------------------------------------------------------------------------------------------------------
def _load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def _cfg(fx, dropout=0.0):
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"], num_attractors=fx["num_attractors"],
                         pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"], dropout=dropout)
    cfg.use_squeezed_transformer = False
    cfg.use_mince_transformer = True
    cfg.mince_scales = list(fx["mince_scales"])
    cfg.mince_channel_props = list(fx["mince_channel_props"])
    cfg.pos_code_type = fx["pos_code_type"]
    cfg.pos_bias_radius = fx["pos_bias_radius"]
    cfg.pos_code_weight = fx["pos_code_weight"]
    cfg.max_pos_size = tuple(fx["grid"])
    return cfg


def _fixture_errors(name):
    fx = _load(name)
    enc = S.SegtranFusionEncoder(_cfg(fx), "Fusion")
    enc.load_state_dict(fx["state_dict"], strict=True)
    enc = enc.to(DEV).eval()
    x = fx["x"].to(DEV).requires_grad_()
    y = enc(x, fx["voxels_pos"].to(DEV), fx["vmask"].to(DEV), torch.Size(fx["grid"]))
    (y * fx["G"].to(DEV)).sum().backward()
    ref = fx["out"]
    e_out = float((y.detach().cpu() - ref).abs().max()) / float(ref.abs().max())
    params = dict(enc.named_parameters())
    gscale = max(float(g.abs().max()) for g in fx["grad_params"].values())
    e_grad = {}
    for k, g in fx["grad_params"].items():
        ours = params[k].grad
        assert ours is not None, k
        # relative to the tensor's own scale, with a floor at the largest gradient's scale (feat2score.bias gradients
        # are zero up to rounding)
        e_grad[k] = float((ours.cpu() - g).abs().max()) / (float(g.abs().max()) + 4e-3 * gscale)
    gx = fx["grad_x"]
    e_grad["x"] = float((x.grad.cpu() - gx).abs().max()) / float(gx.abs().max())
    return fx, e_out, e_grad, enc


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", FIXTURES)
def test_encoder_matches_reference_fixture(name, fused):
    ops.set_attn_fusion(fused)
    try:
        fx, e_out, e_grad, enc = _fixture_errors(name)
    finally:
        ops.set_attn_fusion(True)
    if name == "mince_clamp":
        # scores near 1200 at the first scale saturate its softmax: TF32 operand rounding moves them by ~0.5, which
        # reorders the near-one-hot rows.  The forward stays within the posbias clamp fixture's bound; the gradients are
        # held to the reference in tf32x3 (below), where the products are fp32-grade.
        assert e_out <= 5e-3, e_out
    else:
        assert e_out <= 1e-3, e_out
        worst = max(e_grad, key=e_grad.get)
        assert e_grad[worst] <= 5e-3, (worst, e_grad[worst])
    assert "translayers.0.key.weight" in e_grad and "translayers.0.query.weight" in e_grad       # untied
    if fx["pos_code_type"] == "bias":
        for s in range(len(fx["mince_scales"])):
            assert "pos_code_layers.%d.pos_coder.biases" % s in e_grad
    for layer, mx, cc in zip(enc.translayers, fx["max_attn"], fx["clamp_count"]):
        assert layer.clamp_count == cc
        assert layer.max_attn == pytest.approx(mx, rel=1e-2, abs=1e-4)
        assert layer.lower_clamp_ambiguous_rows == 0


@pytest.mark.parametrize("name", FIXTURES)
def test_encoder_tf32x3_matches_reference_fixture_to_fp32_level(name):
    ops.set_precision("tf32x3")
    try:
        _, e_out, e_grad, _ = _fixture_errors(name)
    finally:
        ops.set_precision("tf32")
    worst = max(e_grad, key=e_grad.get)
    assert e_out < 2e-5, e_out
    assert e_grad[worst] < (1e-3 if name == "mince_clamp" else 1e-4), (worst, e_grad[worst])


def test_encoder_bf16_within_budget():
    # bf16 GEMM operands need 16-byte row pitches: token counts that keep the padded score rows a multiple of 8
    grid, C, scales, props = (8, 8, 8), 64, [1, 2], [1, 1]
    enc = _encoder(grid, [C, C], scales, props).eval()
    B, N = 2, math.prod(grid)
    torch.manual_seed(7)
    x = torch.randn(B, N, C, device=DEV, requires_grad=True)
    vpos, vmask = torch.ones(B, N, 3, device=DEV), torch.ones(B, N, 1, device=DEV)
    gy = torch.randn(B, N, C, device=DEV)
    ops.set_precision("bf16")
    try:
        y = enc(x, vpos, vmask, torch.Size(grid))
        (y * gy).sum().backward()
    finally:
        ops.set_precision("tf32")
    p = {k: v.detach().double().cpu() for k, v in enc.state_dict().items() if v.is_floating_point()}
    x64 = x.detach().double().cpu().requires_grad_()
    y64 = MO.fusion_encoder_mince(p, "", x64, vpos.double().cpu(), vmask.cpu(), [C, C], 4, "bias", grid, scales, props,
                                  pos_bias_radius=2)
    (y64 * gy.double().cpu()).sum().backward()
    e = float((y.detach().double().cpu() - y64.detach()).abs().max() / y64.abs().max())
    ex = float((x.grad.double().cpu() - x64.grad).abs().max() / x64.grad.abs().max())
    assert e < 2e-2 and ex < 5e-2, (e, ex)                 # the budget of tests/test_gpu_bf16.py


# ---------------------------------------------------------------------------------------------------------------------
# a moderate case against the float64 oracle, and training-mode properties
# ---------------------------------------------------------------------------------------------------------------------
def _encoder(grid, dims, scales, props, pos="bias", dropout=0.0, M=4, seed=0):
    torch.manual_seed(seed)
    cfg = encoder_config(S.SegtranConfig, dims=dims, num_modes=M, pos_dim=len(grid), dropout=dropout)
    cfg.use_squeezed_transformer = False
    cfg.use_mince_transformer = True
    cfg.mince_scales, cfg.mince_channel_props = list(scales), list(props)
    cfg.pos_code_type = pos
    cfg.pos_bias_radius = 2
    cfg.max_pos_size = grid
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.init_weights)
    enc.apply(init.tie_qk)
    enc.apply(init.add_identity_bias)
    if pos == "bias":
        with torch.no_grad():
            for layer in enc.pos_code_layers:
                layer.pos_coder.biases.normal_(0, 0.5)
    return enc.to(DEV)


def test_moderate_case_against_float64_oracle():
    grid, C, scales, props = (12, 12, 12), 256, [1, 2, 3], [1, 1, 1]
    enc = _encoder(grid, [C, C], scales, props).eval()
    B, N = 1, math.prod(grid)
    torch.manual_seed(5)
    x = torch.randn(B, N, C, device=DEV, requires_grad=True)
    vpos = torch.ones(B, N, 3, device=DEV)
    vmask = torch.ones(B, N, 1, device=DEV)
    y = enc(x, vpos, vmask, torch.Size(grid))
    gy = torch.randn_like(y)
    (y * gy).sum().backward()
    p = {k: v.detach().double().cpu().requires_grad_() for k, v in enc.state_dict().items() if v.is_floating_point()}
    x64 = x.detach().double().cpu().requires_grad_()
    y64 = MO.fusion_encoder_mince(p, "", x64, vpos.double().cpu(), vmask.cpu(), [C, C], 4, "bias", grid, scales, props,
                                  pos_bias_radius=2)
    assert float((y.detach().double().cpu() - y64.detach()).abs().max()) <= 1e-3 * float(y64.abs().max())
    (y64 * gy.double().cpu()).sum().backward()
    assert float((x.grad.double().cpu() - x64.grad).abs().max()) <= 5e-3 * float(x64.grad.abs().max())
    used = [k for k, _ in enc.named_parameters() if p[k].grad is not None]      # first_norm_layer: no-FFN path only
    gscale = max(float(p[k].grad.abs().max()) for k in used)
    for k, prm in enc.named_parameters():
        g64 = p[k].grad
        if g64 is None:
            assert prm.grad is None, k
            continue
        # relative to the tensor's own scale, floored at the largest gradient's (key.bias gradients are zero up to
        # rounding: a per-query constant does not change a softmax row)
        err = float((prm.grad.double().cpu() - g64).abs().max()) / (float(g64.abs().max()) + 4e-3 * gscale)
        assert err <= 5e-3, (k, err)


def _train_step(enc, grid, B, C, seed=11):
    torch.manual_seed(seed)
    N = math.prod(grid)
    x = torch.randn(B, N, C, device=DEV, requires_grad=True)
    y = enc(x, torch.ones(B, N, len(grid), device=DEV), torch.ones(B, N, 1, device=DEV), torch.Size(grid))
    gy = torch.randn_like(y)
    for p in enc.parameters():
        p.grad = None
    (y * gy).sum().backward()
    # first_norm_layer belongs to the no-FFN path only (reference :456), as without mince
    missing = [n for n, p in enc.named_parameters() if p.grad is None and "first_norm_layer" not in n]
    assert not missing, missing
    return [y.detach(), x.grad.detach()] + [p.grad.detach().clone() for p in _used(enc)]


def _used(enc):
    return [p for n, p in enc.named_parameters() if "first_norm_layer" not in n]


def test_training_step_is_bit_identical_across_runs():
    grid = (8, 9)
    enc = _encoder(grid, [32, 32, 32], [4, 2, 1], [1, 1, 2]).train()
    a = _train_step(enc, grid, 2, 32)
    b = _train_step(enc, grid, 2, 32)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_direct_accumulation_gives_plain_gradients():
    grid = (5, 6, 7)
    enc = _encoder(grid, [32, 32], [1, 2], [1, 1]).train()
    ref = _train_step(enc, grid, 2, 32)[2:]
    for p in enc.parameters():
        p.grad = torch.zeros_like(p)
    ops.set_grad_sink(True)
    try:
        torch.manual_seed(11)
        N = math.prod(grid)
        x = torch.randn(2, N, 32, device=DEV, requires_grad=True)
        y = enc(x, torch.ones(2, N, 3, device=DEV), torch.ones(2, N, 1, device=DEV), torch.Size(grid))
        (y * torch.randn_like(y)).sum().backward()
    finally:
        ops.set_grad_sink(False)
    for p, g in zip(_used(enc), ref):
        assert torch.equal(p.grad, g)


def _graph_step(enc, grid):
    N = math.prod(grid)
    x = torch.randn(2, N, 32, device=DEV, requires_grad=True)
    pos, vm = torch.ones(2, N, 3, device=DEV), torch.ones(2, N, 1, device=DEV)
    params = _used(enc)

    def step():
        for p in params:
            p.grad = None
        x.grad = None
        y = enc(x, pos, vm, torch.Size(grid))
        y.sum().backward()
        return [y, x.grad] + [p.grad for p in params]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step()
    return g, outs, step


def test_cuda_graph_training_step_replays_like_eager():
    grid = (5, 6, 7)
    enc = _encoder(grid, [32, 32, 32], [1, 2], [3, 1]).train()
    g, outs, step = _graph_step(enc, grid)
    g.replay()
    torch.cuda.synchronize()
    got = [t.detach().clone() for t in outs]
    eager = step()
    torch.cuda.synchronize()
    for u, v in zip(got, eager):
        assert torch.equal(u, v.detach())


def test_cuda_graph_replay_with_dropout_is_reproducible():
    grid = (5, 6, 7)
    enc = _encoder(grid, [32, 32, 32], [1, 2], [3, 1], dropout=0.1).train()
    g, outs, _ = _graph_step(enc, grid)
    runs = []
    for base in (1234, 1234, 99):
        ops.reseed(base)
        g.replay()
        torch.cuda.synchronize()
        runs.append([t.detach().clone() for t in outs])
    for u, v in zip(runs[0], runs[1]):
        assert torch.equal(u, v)
    assert not torch.equal(runs[0][0], runs[2][0])          # a new base seed draws new masks
    for t in runs[0][2:]:
        assert torch.isfinite(t).all()


# ---------------------------------------------------------------------------------------------------------------------
# shells: --mince --nosqueeze --pos bias through Segtran3d / Segtran2d with a stand-in backbone (tests/test_gpu_shells.py)
# ---------------------------------------------------------------------------------------------------------------------
def _mince_shell(kind):
    from argparse import Namespace
    from tests.helpers import load_golden
    from tests.test_gpu_shells import FixedFeat2d, FixedFeat3d
    fx = load_golden("seg3d_tiny" if kind == 3 else "seg2d_tiny")
    args = Namespace(**fx["args"])
    args.device = "cuda"
    args.use_squeezed_transformer = False
    args.use_mince_transformer = True
    args.mince_scales = [1, 2]
    args.mince_channel_props = [1, 1]
    args.pos_code_type = "bias"
    args.pos_bias_radius = 1
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    feats = [f.cuda().requires_grad_(i > 0) for i, f in enumerate(fx["feats"])]
    if kind == 3:
        import segtran_b200.networks.segtran3d as M
        cfg = M.Segtran3dConfig()
        cfg.update_config(args)
        net = M.Segtran3d(cfg, backbone=FixedFeat3d(feats))
    else:
        import segtran_b200.networks.segtran2d as M
        cfg = M.Segtran2dConfig()
        cfg.update_config(args)
        net = M.Segtran2d(cfg, backbone=FixedFeat2d(feats))
    return fx, net.cuda().train(), feats


@pytest.mark.parametrize("kind", [3, 2])
def test_shells_run_mince_forward_and_backward(kind):
    fx, net, feats = _mince_shell(kind)
    assert isinstance(net.voxel_fusion.translayers[0], S.CrossMinceAttFeatTrans)
    with torch.no_grad():
        for layer in net.voxel_fusion.pos_code_layers:
            layer.pos_coder.biases.normal_(0, 0.5)
    y = net(fx["batch"].cuda())
    y.float().sum().backward()
    assert torch.isfinite(y).all()
    for s, layer in enumerate(net.voxel_fusion.pos_code_layers):
        g = layer.pos_coder.biases.grad
        assert g is not None and torch.isfinite(g).all() and float(g.abs().max()) > 0, s
    assert net.voxel_fusion.translayers[0].key.weight.grad is not None
