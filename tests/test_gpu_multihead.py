"""The multi-head ablation (--nosqueeze --multihead, MultiHeadFeatTrans) on the GPU: parity with the reference's fixtures
(oracle/gen_multihead_golden.py) on both attention paths and in every precision mode, the Segtran3d / Segtran2d shells,
full-size stacks against the fp32 oracle, the two dropout sites, run-to-run bit identity, direct gradient accumulation
and CUDA-graph replay of a training step."""
import math
import os
from argparse import Namespace

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import segtran_b200.networks.segtran_shared as S  # noqa: E402
from oracle import multihead_oracle as MH  # noqa: E402
from oracle import segtran_oracle as O  # noqa: E402
from segtran_b200 import ops, train  # noqa: E402
from segtran_b200.graph import CapturedStep  # noqa: E402
from tests.helpers import encoder_config, load_golden, rel_err, rms_rel  # noqa: E402
from tests.test_multihead_cpu import NAMES, mh_cfg  # noqa: E402

DEV = "cuda"
# (forward, gradient) tolerances, max|a-b|/max|b|; gradients are floored at 4e-3 of the largest gradient in the model
TOL = {"tf32": (1e-3, 5e-3), "tf32x3": (1e-5, 1e-4), "bf16": (2e-2, 2e-2)}
# multihead_clamp's scores reach ~7000.  A softmax over saturated scores amplifies operand rounding (as for posbias_clamp
# in tests/test_gpu_posbias.py): TF32 operands get that fixture's bounds; in tf32x3 the reference's own float32 rounding
# (2e-5 on the output, 1e-3 on gradients, see tests/test_multihead_cpu.py) is the limit
CLAMP_TOL = {"tf32": (5e-3, 5e-2), "tf32x3": (3e-5, 1e-3)}


@pytest.fixture
def precision():
    old = ops.get_precision()
    yield ops.set_precision
    ops.set_precision(old)


@pytest.fixture
def fusion():
    old = ops._ATTN_FUSION
    yield ops.set_attn_fusion
    ops.set_attn_fusion(old)


def _fixture_encoder(fx):
    cfg = mh_cfg(fx)
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    enc.apply(S.SegtranInitWeights(cfg).tie_qk)
    enc.load_state_dict(fx["state_dict"], strict=True)
    return enc.to(DEV).eval()


def _fixture_loss(fx, enc, x):
    y = enc(x, fx["voxels_pos"].to(DEV), fx["vmask"].to(DEV), torch.Size(fx["grid"]))
    if fx["use_attn_consist_loss"]:
        fun = train.attn_consist_loss3d if fx["three_d"] else train.attn_consist_loss2d
        return y, fun(enc.layers_attn_scores, torch.Size(fx["grid"]), fx["seg_mask"].to(DEV))
    return y, (y * fx["G"].to(DEV)).sum()


def _check_grads(named_params, grad_ref, tol):
    gscale = max(float(g.abs().max()) for g in grad_ref.values())
    for k, gref in grad_ref.items():
        ours = named_params[k].grad
        if float(gref.abs().max()) == 0.0:
            assert ours is None or float(ours.abs().max()) <= 1e-5 * gscale, k
            continue
        assert ours is not None, k
        err = float((ours.cpu() - gref).abs().max()) / (float(gref.abs().max()) + 4e-3 * gscale)
        assert err <= tol, (k, err)


CASES = [(n, "tf32", f) for n in NAMES for f in (True, False)] + [(n, "tf32x3", False) for n in NAMES] + \
    [("multihead_2d", "bf16", True), ("multihead_2d", "bf16", False)]


@pytest.mark.parametrize("name,prec,fused", CASES)
def test_encoder_matches_reference_fixture(name, prec, fused, precision, fusion):
    precision(prec)
    fusion(fused)
    fx = load_golden(name)
    enc = _fixture_encoder(fx)
    x = fx["x"].to(DEV).requires_grad_()
    y, loss = _fixture_loss(fx, enc, x)
    loss.backward()
    fwd_tol, grad_tol = CLAMP_TOL[prec] if name == "multihead_clamp" else TOL[prec]
    e = rel_err(y, fx["out"])
    print("%s %s fused=%s: out %.2e dx %.2e" % (name, prec, fused, e, rel_err(x.grad, fx["grad_x"])))
    assert e <= fwd_tol
    if fx["use_attn_consist_loss"]:
        assert abs(float(loss.detach()) - float(fx["loss"])) <= fwd_tol * abs(float(fx["loss"]))
    assert rel_err(x.grad, fx["grad_x"]) <= grad_tol
    _check_grads(dict(enc.named_parameters()), fx["grad_params"], grad_tol)
    for layer, m in zip(enc.translayers, fx["max_attn"]):
        assert layer.max_attn == pytest.approx(m, rel=1e-2)
    if name == "multihead_clamp":
        assert enc.translayers[0].clamp_count == 1 and enc.translayers[0].lower_clamp_ambiguous_rows == 0


# ---------------------------------------------------------------------------------------------------------------------
# shells: Segtran3d / Segtran2d with --nosqueeze --multihead on a fixed-feature backbone
# ---------------------------------------------------------------------------------------------------------------------
def _shell(kind):
    from tests.test_gpu_shells import FixedFeat2d, FixedFeat3d
    fx = load_golden("multihead_seg3d" if kind == 3 else "multihead_seg2d")
    inp = load_golden(fx["inputs"])
    args = Namespace(**fx["args"])
    args.device = "cuda"
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    feats = [f.cuda().requires_grad_(i > 0) for i, f in enumerate(inp["feats"])]
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
    missing, unexpected = net.load_state_dict(fx["state_dict"], strict=False)
    assert not unexpected and not missing, (missing, unexpected)
    return fx, inp, net.cuda().eval(), feats


def _sampled_err(t, ref):
    """max|a-b| over the fixture's sampled elements / max|b| over the whole reference tensor (oracle/gen_multihead_golden.py)."""
    assert tuple(t.shape) == ref["shape"]
    got = t.detach().reshape(-1)[ref["idx"].long().to(t.device)].double().cpu()
    return float((got - ref["val"].double()).abs().max()) / ref["absmax"]


@pytest.mark.parametrize("kind", [3, 2])
def test_shell_matches_reference_fixture(kind):
    fx, inp, net, feats = _shell(kind)
    assert all(isinstance(t.out_trans, S.MultiHeadFeatTrans) for t in net.voxel_fusion.translayers)
    y = net(inp["batch"].cuda())
    e = _sampled_err(y, fx["out"])
    (y * inp["G"].cuda()).sum().backward()
    print("multihead seg%dd: logits %.2e" % (kind, e))
    assert e <= 1e-3
    for i in range(1, 5):
        assert _sampled_err(feats[i].grad, fx["grad_feats"][i]) <= 5e-3, i
    grads = {k: g for k, g in fx["grad_params"].items() if not k.startswith("backbone.")}
    _check_grads(dict(net.named_parameters()), grads, 5e-3)


# ---------------------------------------------------------------------------------------------------------------------
# full-size stacks against the fp32 oracle (cfg-1 and cfg-4 shapes of tests/test_gpu_fullsize_configs.py)
# ---------------------------------------------------------------------------------------------------------------------
FULL = {1: ([1792, 1792], (36, 36), 2), 4: ([1024, 1024], (14, 14, 14), 4)}


def _mh_encoder(dims, grid, seed, dropout=0.0, out_type="private"):
    cfg = encoder_config(S.SegtranConfig, dims=dims, num_modes=4, num_attractors=16, pos_dim=len(grid), dropout=dropout)
    cfg.use_squeezed_transformer = False
    cfg.ablate_multihead = True
    cfg.trans_output_type = out_type
    torch.manual_seed(seed)
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.init_weights)
    enc.apply(init.tie_qk)
    enc.apply(init.add_identity_bias)
    return enc


@pytest.mark.parametrize("cfg", [1, 4])
def test_full_size_stack_against_oracle(cfg):
    dims, grid, B = FULL[cfg]
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    enc = _mh_encoder(dims, grid, seed=80 + cfg).eval()
    p = {k: v.clone().requires_grad_() for k, v in enc.state_dict().items() if ".key." not in k}
    N = math.prod(grid)
    torch.manual_seed(cfg)
    x = torch.randn(B, N, dims[0]) * 1.5 + 0.2
    pos = O.voxels_pos_for_grid(grid, (8,) * len(grid), B)
    mask = (torch.rand(B, N, 1) > 0.05).float() if len(grid) == 2 else torch.ones(B, N, 1)
    G = torch.randn(B, N, dims[-1])
    xr = x.clone().requires_grad_()
    ref = MH.fusion_encoder_multihead(p, "", xr, pos, mask, dims, 4)
    (ref * G).sum().backward()
    enc = enc.cuda()
    xg = x.cuda().requires_grad_()
    y = enc(xg, pos.cuda(), mask.cuda(), torch.Size(grid))
    (y * G.cuda()).sum().backward()
    e, r, ex = rel_err(y, ref), rms_rel(y, ref), rel_err(xg.grad, xr.grad)
    print("multihead cfg%d N=%d B=%d: fwd max-rel %.2e rms-rel %.2e | dx max-rel %.2e" % (cfg, N, B, e, r, ex))
    assert e < 1e-3 and ex < 3e-3
    got = dict(enc.named_parameters())
    gscale = max(float(v.grad.abs().max()) for v in p.values() if v.grad is not None)
    for k, v in p.items():
        gm = float(v.grad.abs().max())
        err = float((got[k].grad.cpu() - v.grad).abs().max())
        assert err <= 5e-3 * gm + 1e-6 * gscale, (k, err, gm, gscale)
    assert enc.translayers[0].lower_clamp_ambiguous_rows == 0


# ---------------------------------------------------------------------------------------------------------------------
# dropout: the output Linear's epilogue (after bias and residual) and the attention probabilities
# ---------------------------------------------------------------------------------------------------------------------
def test_output_dropout_keep_rate_and_backward_mask():
    torch.manual_seed(1)
    R, I, O_ = 4096, 96, 64
    g = torch.randn(R, I, device=DEV, requires_grad=True)
    W = torch.randn(O_, I, 1, device=DEV, requires_grad=True)           # a Conv1d weight, read as [O, I]
    b = torch.randn(O_, device=DEV, requires_grad=True)
    u = (torch.randn(R, O_, device=DEV) + 3.0).requires_grad_()           # residual, never 0
    p = 0.3
    z = ops.linear(g, W, b, drop_p=p, seed=ops.new_dropout_seed(torch.device(DEV)), tag="proj", round_out=False, addend=u)
    kept = z != 0
    rate = float(kept.float().mean())
    assert abs(rate - (1 - p)) < 0.01, rate
    ref = (g @ W[..., 0].t() + b + u) / (1 - p)                            # the residual is dropped with the sum
    assert float((z.detach() - ref)[kept].abs().max()) <= 2e-3 * float(ref.abs().max())
    z.backward(torch.ones_like(z))
    # d z / d u = keep / (1 - p): the backward regenerates the forward's mask
    assert torch.equal(u.grad != 0, kept)
    assert torch.allclose(u.grad[kept], torch.full_like(u.grad[kept], 1 / (1 - p)), rtol=1e-3)     # TF32-rounded
    assert torch.allclose(b.grad, u.grad.sum(0), rtol=1e-5)


def test_attention_dropout_keep_rate_and_backward_mask():
    torch.manual_seed(2)
    B, M, N, d = 2, 4, 200, 8
    q = ops.round_tf32(torch.randn(B, N, M * d, device=DEV)).requires_grad_()
    k = ops.round_tf32(torch.randn(B, N, M * d, device=DEV)).requires_grad_()
    p = 0.25
    P = ops.attn_probs(q, k, M, 1 / math.sqrt(d), 500.0, p, ops.new_dropout_seed(torch.device(DEV)))
    kept = P != 0
    rate = float(kept.float().mean())
    assert abs(rate - (1 - p)) < 0.01, rate
    dP = torch.randn_like(P)
    P.backward(dP)
    q64, k64 = q.detach().double().requires_grad_(), k.detach().double().requires_grad_()
    s = torch.einsum("bumd,bvmd->bmuv", q64.view(B, N, M, d), k64.view(B, N, M, d)) / math.sqrt(d)
    P64 = torch.softmax(s, -1) * kept / (1 - p)
    assert rel_err(P, P64) <= 1e-3
    (P64 * dP.double()).sum().backward()
    assert rel_err(q.grad, q64.grad) <= 5e-3 and rel_err(k.grad, k64.grad) <= 5e-3


def test_training_layer_with_both_dropout_sites():
    grid = (6, 7)
    enc = _mh_encoder([64, 64], grid, seed=3, dropout=0.2).to(DEV).train()
    N = math.prod(grid)
    x = torch.randn(2, N, 64, device=DEV, requires_grad=True)
    y = enc(x, torch.ones(2, N, 2, device=DEV), torch.ones(2, N, 1, device=DEV), torch.Size(grid))
    y.sum().backward()
    assert torch.isfinite(y).all() and torch.isfinite(x.grad).all()
    missing = [n for n, prm in enc.named_parameters() if prm.grad is None]
    assert not missing, missing


# ---------------------------------------------------------------------------------------------------------------------
# training-mode properties
# ---------------------------------------------------------------------------------------------------------------------
def _train_step(enc, grid, x, gy):
    for prm in enc.parameters():
        prm.grad = None
    x.grad = None
    N = math.prod(grid)
    y = enc(x, torch.ones(x.shape[0], N, len(grid), device=DEV), torch.ones(x.shape[0], N, 1, device=DEV),
            torch.Size(grid))
    (y * gy).sum().backward()
    return [y.detach().clone(), x.grad.detach().clone()] + [prm.grad.detach().clone() for prm in enc.parameters()]


@pytest.mark.parametrize("out_type,dims", [("private", [64, 64, 32]), ("shared", [36, 36])])
def test_training_step_is_bit_identical_across_runs(out_type, dims):
    grid = (5, 6, 7)
    enc = _mh_encoder(dims, grid, seed=4, out_type=out_type).to(DEV).train()
    torch.manual_seed(5)
    x = torch.randn(2, math.prod(grid), dims[0], device=DEV, requires_grad=True)
    gy = torch.randn(2, math.prod(grid), dims[-1], device=DEV)
    a = _train_step(enc, grid, x, gy)
    b = _train_step(enc, grid, x, gy)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_direct_accumulation_gives_plain_gradients():
    grid = (5, 6, 7)
    for out_type in ("private", "shared"):
        enc = _mh_encoder([64, 64], grid, seed=6, out_type=out_type).to(DEV).train()
        x = torch.randn(2, math.prod(grid), 64, device=DEV, requires_grad=True)
        gy = torch.randn(2, math.prod(grid), 64, device=DEV)
        ref = _train_step(enc, grid, x, gy)[2:]
        for prm in enc.parameters():
            prm.grad = torch.zeros_like(prm)
        ops.set_grad_sink(True)
        try:
            N = math.prod(grid)
            y = enc(x, torch.ones(2, N, 3, device=DEV), torch.ones(2, N, 1, device=DEV), torch.Size(grid))
            (y * gy).sum().backward()
        finally:
            ops.set_grad_sink(False)
        for prm, g in zip(enc.parameters(), ref):
            assert torch.equal(prm.grad, g)


def _captured(enc, grid, C):
    N = math.prod(grid)
    x = torch.randn(2, N, C, device=DEV, requires_grad=True)
    pos, vm = torch.ones(2, N, len(grid), device=DEV), torch.ones(2, N, 1, device=DEV)
    params = list(enc.parameters())

    def step():
        for prm in params:
            prm.grad = None
        x.grad = None
        y = enc(x, pos, vm, torch.Size(grid))
        y.sum().backward()
        return [y, x.grad] + [prm.grad for prm in params]

    return CapturedStep(step, warmup=2), step


def test_cuda_graph_training_step_replays_like_eager():
    grid = (5, 6, 7)
    enc = _mh_encoder([64, 64, 32], grid, seed=7).to(DEV).train()
    graph, step = _captured(enc, grid, 64)
    outs = graph()
    torch.cuda.synchronize()
    got = [t.detach().clone() for t in outs]
    eager = step()
    torch.cuda.synchronize()
    for u, v in zip(got, eager):
        assert torch.equal(u, v.detach())


def test_cuda_graph_replay_with_dropout_is_reproducible():
    grid = (5, 6, 7)
    enc = _mh_encoder([64, 64], grid, seed=8, dropout=0.1).to(DEV).train()
    graph, _ = _captured(enc, grid, 64)
    runs = []
    for base in (1234, 1234, 99):
        ops.reseed(base)
        outs = graph()
        torch.cuda.synchronize()
        runs.append([t.detach().clone() for t in outs])
    for u, v in zip(runs[0], runs[1]):
        assert torch.equal(u, v)
    assert not torch.equal(runs[0][0], runs[2][0])
    for t in runs[0][2:]:
        assert torch.isfinite(t).all()
