"""Sliding-window positional biases (--pos bias) and the prologue without a positional code (--pos none) on the GPU,
against a float64 PyTorch restatement of the reference's dense [N,N] bias (segtran_shared.py:1002-1175, :578-605)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from segtran_b200 import ops  # noqa: E402
import segtran_b200.networks.segtran_shared as S  # noqa: E402
from tests.helpers import encoder_config  # noqa: E402

DEV = "cuda"


def dense_bias(table, R, grid):
    """[N,N] float64: bias[q,k] = table[k - q + R] inside the window, 0 outside (the reference's expanded matrix)."""
    axes = [torch.arange(g) for g in grid]
    c = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1).reshape(-1, len(grid))
    diff = c[None, :, :] - c[:, None, :]                      # k - q, [q, k, pd]
    inwin = (diff.abs() <= R).all(-1)
    idx = (diff + R).clamp(0, 2 * R)
    vals = table.double().cpu()[tuple(idx[..., i] for i in range(len(grid)))]
    return torch.where(inwin, vals, torch.zeros((), dtype=torch.float64))


def ref_softmax(S64, table64, R, grid, w, clip):
    """float64 restatement: clamp decided on the raw max, then + w*bias, then softmax (no dropout)."""
    Sc = S64.clamp(-clip, clip) if float(S64.max()) > clip else S64
    return torch.softmax(Sc + w * dense_bias(table64, R, grid).to(S64), dim=-1)


CASES = [((5, 6, 7), 2, 1.0, 2), ((6, 7), 2, 0.5, 1), ((3, 4, 5), 1, 1.5, 1)]


@pytest.mark.parametrize("grid,R,w,B", CASES)
def test_unfused_softmax_with_posbias_and_table_gradient(grid, R, w, B):
    torch.manual_seed(0)
    N, M = math.prod(grid), 2
    table = (torch.randn([2 * R + 1] * len(grid)) * 0.7).to(DEV).requires_grad_()
    s = (torch.randn(B, M, N, N) * 3).to(DEV).requires_grad_()
    g = torch.randn(B, M, N, N, device=DEV)
    amax = s.detach().max().reshape(1)
    P = ops.softmax(s, amax, 500.0, posbias=ops.PosBias(table, R, grid, w))
    (P * g).sum().backward()
    s64 = s.detach().double().cpu().requires_grad_()
    t64 = table.detach().double().cpu().requires_grad_()
    Pr = ref_softmax(s64, t64, R, grid, w, 500.0)
    (Pr * g.double().cpu()).sum().backward()
    torch.testing.assert_close(P.detach().cpu().double(), Pr.detach(), rtol=2e-3, atol=1e-6)
    torch.testing.assert_close(s.grad.cpu().double(), s64.grad, rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(table.grad.cpu().double(), t64.grad, rtol=1e-3, atol=1e-4)


def test_softmax_clamp_then_bias_and_gradient_before_the_clamp_mask():
    torch.manual_seed(1)
    grid, R, w, clip = (5, 6, 7), 2, 1.0, 5.0
    N = math.prod(grid)
    table = torch.randn([2 * R + 1] * 3).to(DEV).requires_grad_()
    s = (torch.randn(1, 1, N, N) * 8).to(DEV).requires_grad_()     # many scores beyond +-clip
    g = torch.randn(1, 1, N, N, device=DEV)
    amax = s.detach().max().reshape(1)
    assert float(amax) > clip
    P = ops.softmax(s, amax, clip, posbias=ops.PosBias(table, R, grid, w))
    (P * g).sum().backward()
    s64 = s.detach().double().cpu().requires_grad_()
    t64 = table.detach().double().cpu().requires_grad_()
    # the table sees dS' of every element, clamped or not: restate it with the clamp's value but an identity gradient
    sc = s64 + (s64.clamp(-clip, clip) - s64).detach()
    Pr = torch.softmax(sc + w * dense_bias(t64, R, grid), -1)
    (Pr * g.double().cpu()).sum().backward()
    torch.testing.assert_close(P.detach().cpu().double(), Pr.detach(), rtol=2e-3, atol=1e-6)
    torch.testing.assert_close(table.grad.cpu().double(), t64.grad, rtol=1e-3, atol=1e-4)
    # dS itself carries the clamp mask
    inside = (s64.detach().abs() <= clip)
    torch.testing.assert_close(s.grad.cpu().double(), s64.grad * inside, rtol=5e-3, atol=1e-5)


@pytest.mark.parametrize("grid,R,w,B", CASES)
def test_fused_probabilities_match_restatement_and_unfused_softmax(grid, R, w, B):
    torch.manual_seed(2)
    N, M, d = math.prod(grid), 4, 16
    table = (torch.randn([2 * R + 1] * len(grid)) * 0.7).to(DEV)
    q = ops.round_tf32(torch.randn(B, N, M * d, device=DEV))
    k = ops.round_tf32(torch.randn(B, N, M * d, device=DEV))
    pb = ops.PosBias(table, R, grid, w)
    P, Sraw, lse, rowmax, stat = ops.attn_probs_fused(q, k, M, 500.0, need_scores=True, round_out=False, posbias=pb)
    q64 = q.double().cpu().view(B, N, M, d).permute(0, 2, 1, 3)
    k64 = k.double().cpu().view(B, N, M, d).permute(0, 2, 1, 3)
    s64 = q64 @ k64.transpose(-1, -2) / math.sqrt(d)
    Pr = ref_softmax(s64, table, R, grid, w, 500.0)
    torch.testing.assert_close(P.cpu().double(), Pr, rtol=2e-3, atol=2e-6)
    # S and rowmax stay raw; lse is the biased row's
    torch.testing.assert_close(Sraw.cpu().double(), s64, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(rowmax.cpu().double(), s64.amax(-1), rtol=1e-4, atol=1e-4)
    biased = s64 + w * dense_bias(table, R, grid)
    torch.testing.assert_close(lse.cpu().double(), torch.logsumexp(biased, -1), rtol=1e-4, atol=1e-4)
    # the unfused kernel on the same raw scores
    Pu = ops.softmax(Sraw, stat[2:], 500.0, posbias=pb)
    torch.testing.assert_close(P, Pu.detach(), rtol=1e-3, atol=1e-6)


def test_fused_clamp_case():
    torch.manual_seed(3)
    grid, R, M, d, B = (5, 6, 7), 2, 2, 16, 1
    N = math.prod(grid)
    table = torch.randn([2 * R + 1] * 3).to(DEV)
    q = ops.round_tf32(torch.randn(B, N, M * d, device=DEV) * 12)
    k = ops.round_tf32(torch.randn(B, N, M * d, device=DEV) * 12)
    diag = torch.tensor([-3.0e38, 0.0, 0.0], device=DEV)
    P, Sraw, _, _, _ = ops.attn_probs_fused(q, k, M, 500.0, diag=diag, need_scores=True, round_out=False,
                                            posbias=ops.PosBias(table, R, grid, 1.0))
    s64 = Sraw.cpu().double()
    assert float(s64.max()) > 500.0
    torch.testing.assert_close(P.cpu().double(), ref_softmax(s64, table, R, grid, 1.0, 500.0), rtol=2e-3, atol=2e-6)
    assert float(diag[1]) == 1.0 and float(diag[2]) == 0.0


def test_prologue_without_positional_code():
    torch.manual_seed(4)
    B, N, C = 2, 45, 36
    x = torch.randn(B, N, C, device=DEV, requires_grad=True)
    g = (1 + 0.1 * torch.randn(C, device=DEV)).requires_grad_()
    b = (0.1 * torch.randn(C, device=DEV)).requires_grad_()
    mask = (torch.rand(B * N, device=DEV) > 0.2).float()
    dh = torch.randn(B, N, C, device=DEV)
    h = ops.prologue(x, g, b, None, 0.0, mask, 0.0, 0)
    (h * dh).sum().backward()
    x64, g64, b64 = (t.detach().double().cpu().requires_grad_() for t in (x, g, b))
    h64 = torch.nn.functional.layer_norm(x64, (C,), g64, b64, eps=1e-12) * mask.double().cpu().view(B, N, 1)
    (h64 * dh.double().cpu()).sum().backward()
    torch.testing.assert_close(h.detach().cpu().double(), h64.detach(), rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(x.grad.cpu().double(), x64.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(g.grad.cpu().double(), g64.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(b.grad.cpu().double(), b64.grad, rtol=1e-4, atol=1e-4)


def test_prologue_without_code_dropout_masks_agree():
    torch.manual_seed(5)
    B, N, C = 2, 30, 32
    x = torch.randn(B, N, C, device=DEV, requires_grad=True)
    g = torch.ones(C, device=DEV, requires_grad=True)
    b = torch.zeros(C, device=DEV, requires_grad=True)
    seed = ops.new_dropout_seed(x.device)
    h = ops.prologue(x, g, b, None, 0.0, None, 0.3, seed)
    h.sum().backward()
    dropped = h.detach() == 0
    assert 0.2 < float(dropped.float().mean()) < 0.4
    # d h / d b = keep mask * 1/(1-p) per element: its column sums count the kept elements
    kept = (~dropped).float().sum((0, 1)) / 0.7
    torch.testing.assert_close(b.grad, kept, rtol=1e-5, atol=1e-4)


def _bias_encoder(grid, dims, seed=0, w=1.0, dropout=0.0):
    torch.manual_seed(seed)
    cfg = encoder_config(S.SegtranConfig, dims=dims, num_modes=4, pos_dim=len(grid), dropout=dropout)
    cfg.use_squeezed_transformer = False
    cfg.pos_code_type = "bias"
    cfg.pos_bias_radius = 2
    cfg.pos_code_weight = w
    cfg.max_pos_size = grid
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.init_weights)
    enc.apply(init.tie_qk)
    enc.apply(init.add_identity_bias)
    with torch.no_grad():
        enc.pos_code_layer.pos_coder.biases.normal_(0, 0.5)
    return enc.to(DEV)


def _run(enc, grid, B, C, seed=11):
    torch.manual_seed(seed)
    N = math.prod(grid)
    x = torch.randn(B, N, C, device=DEV, requires_grad=True)
    pos = torch.ones(B, N, len(grid), device=DEV)
    vmask = torch.ones(B, N, 1, device=DEV)
    y = enc(x, pos, vmask, torch.Size(grid))
    gy = torch.randn_like(y)
    for p in enc.parameters():
        p.grad = None
    (y * gy).sum().backward()
    return y.detach(), x.grad.detach(), enc.pos_code_layer.pos_coder.biases.grad.detach().clone()


@pytest.mark.parametrize("grid,B", [((5, 6, 7), 2), ((6, 7), 1)])
def test_encoder_fused_matches_unfused_and_fp32_products(grid, B):
    enc = _bias_encoder(grid, [32, 32, 32], w=0.5)
    y_f, dx_f, dT_f = _run(enc, grid, B, 32)
    ops.set_attn_fusion(False)
    try:
        y_u, dx_u, dT_u = _run(enc, grid, B, 32)
    finally:
        ops.set_attn_fusion(True)
    ops.set_precision("tf32x3")
    try:
        y_x, dx_x, dT_x = _run(enc, grid, B, 32)
    finally:
        ops.set_precision("tf32")
    assert float(dT_x.abs().max()) > 0
    for a in (y_f, y_u):
        torch.testing.assert_close(a, y_x, rtol=0, atol=1e-2)
    # each softmax row's dS' sums to zero, so the table gradient is a small difference of O(1e-3)-accurate TF32 terms;
    # its float64 accuracy is checked per kernel above, here it only has to agree between the paths at that level
    torch.testing.assert_close(dT_f, dT_u, rtol=0, atol=0.1 * float(dT_x.abs().max()))
    for a in (dT_f, dT_u):
        torch.testing.assert_close(a, dT_x, rtol=0, atol=0.3 * float(dT_x.abs().max()))
    for a in (dx_f, dx_u):
        torch.testing.assert_close(a, dx_x, rtol=0, atol=2e-2 * float(dx_x.abs().max()))


def test_table_gradient_is_bit_identical_across_runs():
    grid = (5, 6, 7)
    enc = _bias_encoder(grid, [32, 32, 32])
    a = _run(enc, grid, 2, 32)
    b = _run(enc, grid, 2, 32)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_direct_accumulation_gives_plain_gradients():
    grid = (6, 7)
    enc = _bias_encoder(grid, [32, 32, 32])
    _, _, dT = _run(enc, grid, 2, 32)
    tbl = enc.pos_code_layer.pos_coder.biases
    tbl.grad = torch.zeros_like(tbl)
    ops.set_grad_sink(True)
    try:
        torch.manual_seed(11)
        N = math.prod(grid)
        x = torch.randn(2, N, 32, device=DEV, requires_grad=True)
        y = enc(x, torch.ones(2, N, 2, device=DEV), torch.ones(2, N, 1, device=DEV), torch.Size(grid))
        (y * torch.randn_like(y)).sum().backward()
    finally:
        ops.set_grad_sink(False)
    assert torch.equal(tbl.grad, dT)


def test_eval_mode_caches_a_table_snapshot():
    grid = (6, 7)
    enc = _bias_encoder(grid, [32, 32]).eval()
    N = math.prod(grid)
    x = torch.randn(1, N, 32, device=DEV)
    pos, vm = torch.ones(1, N, 2, device=DEV), torch.ones(1, N, 1, device=DEV)
    with torch.no_grad():
        y0 = enc(x, pos, vm, torch.Size(grid))
        enc.pos_code_layer.pos_coder.biases.add_(1.0)      # the reference keeps its cached bias matrix for this shape
        y1 = enc(x, pos, vm, torch.Size(grid))
    assert torch.equal(y0, y1)


def test_cuda_graph_training_step_replays_like_eager():
    grid = (5, 6, 7)
    enc = _bias_encoder(grid, [32, 32, 32]).train()
    N = math.prod(grid)
    x = torch.randn(2, N, 32, device=DEV, requires_grad=True)
    pos, vm = torch.ones(2, N, 3, device=DEV), torch.ones(2, N, 1, device=DEV)
    tbl = enc.pos_code_layer.pos_coder.biases

    def step():
        tbl.grad = None
        x.grad = None
        y = enc(x, pos, vm, torch.Size(grid))
        y.sum().backward()
        return y, tbl.grad

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y_g, dT_g = step()
    g.replay()
    torch.cuda.synchronize()
    yg, dTg = y_g.detach().clone(), dT_g.clone()
    y_e, dT_e = step()
    torch.cuda.synchronize()
    assert torch.equal(yg, y_e.detach())
    assert torch.equal(dTg, dT_e)


# ---------------------------------------------------------------------------------------------------------------------
# against the fixtures made by the reference (oracle/gen_posbias_golden.py)
# ---------------------------------------------------------------------------------------------------------------------
import os  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = ["posbias3d", "posbias2d", "posnone_sq"]


def _fixture_encoder(fx):
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"], num_attractors=fx["num_attractors"],
                         pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"])
    cfg.use_squeezed_transformer = fx["use_squeezed_transformer"]
    cfg.pos_code_type = fx["pos_code_type"]
    cfg.pos_bias_radius = fx["pos_bias_radius"]
    cfg.pos_code_weight = fx["pos_code_weight"]
    cfg.max_pos_size = tuple(fx["grid"])
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    enc.apply(S.SegtranInitWeights(cfg).tie_qk)
    enc.load_state_dict(fx["state_dict"], strict=True)
    return enc.to(DEV).eval()


def _fixture_errors(name):
    fx = torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)
    enc = _fixture_encoder(fx)
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
        if float(g.abs().max()) == 0.0:           # never-used parameters (the in-squeeze's one-mode aggregate)
            assert ours is None or float(ours.abs().max()) <= 1e-5 * gscale, k
            continue
        assert ours is not None, k
        # relative to the tensor's own scale, with a floor at the largest gradient's scale (feat2score.bias gradients
        # are zero up to rounding)
        e_grad[k] = float((ours.cpu() - g).abs().max()) / (float(g.abs().max()) + 4e-3 * gscale)
    gx = fx["grad_x"]
    e_grad["x"] = float((x.grad.cpu() - gx).abs().max()) / float(gx.abs().max())
    return fx, e_out, e_grad, enc


@pytest.mark.parametrize("name", FIXTURES)
def test_encoder_matches_reference_fixture(name):
    fx, e_out, e_grad, _ = _fixture_errors(name)
    assert e_out <= 1e-3, e_out
    worst = max(e_grad, key=e_grad.get)
    assert e_grad[worst] <= 5e-3, (worst, e_grad[worst])
    if fx["pos_code_type"] == "bias":
        assert "pos_code_layer.pos_coder.biases" in e_grad


@pytest.mark.parametrize("name", FIXTURES)
def test_encoder_tf32x3_matches_reference_fixture_to_fp32_level(name):
    ops.set_precision("tf32x3")
    try:
        _, e_out, e_grad, _ = _fixture_errors(name)
    finally:
        ops.set_precision("tf32")
    worst = max(e_grad, key=e_grad.get)
    assert e_out < 2e-5, e_out
    assert e_grad[worst] < 1e-4, (worst, e_grad[worst])


def test_clamp_then_bias_matches_reference_fixture():
    """Scores up to ~1600 > attn_clip=500: the clamp fires, then the bias is added.  A softmax over saturated scores
    amplifies operand rounding (as for enc3d_clamp in test_gpu_encoder.py), hence its own bounds."""
    fx, e_out, e_grad, enc = _fixture_errors("posbias_clamp")
    t = enc.translayers[0]
    assert t.clamp_count == 1 and abs(t.max_attn - fx["max_attn"][0]) < 1e-2 * fx["max_attn"][0]
    assert t.lower_clamp_ambiguous_rows == 0
    worst = max(e_grad, key=e_grad.get)
    assert e_out <= 5e-3, e_out
    assert e_grad[worst] <= 5e-2, (worst, e_grad[worst])       # TF32 operands through the saturated softmax
    ops.set_precision("tf32x3")                                 # fp32-level products: tight again
    try:
        _, e_out, e_grad, _ = _fixture_errors("posbias_clamp")
    finally:
        ops.set_precision("tf32")
    worst = max(e_grad, key=e_grad.get)
    assert e_out < 2e-5, e_out
    assert e_grad[worst] < 1e-3, (worst, e_grad[worst])


@pytest.mark.parametrize("grid,B", [((5, 6, 7), 2), ((6, 7), 1)])
def test_fused_dropout_mask_and_table_gradient(grid, B):
    """The fused forward's dropout mask is the one the biased softmax backward regenerates, and the table gradient of the
    fused path (the backward ops.softmax_backward runs, through softmax_posbias_backward, on the saved raw scores)
    matches float64 autograd of the restatement."""
    torch.manual_seed(6)
    R, w, M, d, p = 2, 0.7, 4, 16, 0.3
    N = math.prod(grid)
    table = (torch.randn([2 * R + 1] * len(grid)) * 0.7).to(DEV)
    q = ops.round_tf32(torch.randn(B, N, M * d, device=DEV))
    k = ops.round_tf32(torch.randn(B, N, M * d, device=DEV))
    seed = 987654321
    P, Sraw, lse, _, stat = ops.attn_probs_fused(q, k, M, 500.0, drop_p=p, seed=seed, need_scores=True, round_out=False,
                                                 posbias=ops.PosBias(table, R, grid, w))
    keep = (P != 0).cpu()
    assert 0.25 < 1 - float(keep.double().mean()) < 0.35
    g = torch.randn(B, M, N, N, device=DEV)
    dP = torch.empty_strided(P.size(), P.stride(), device=DEV)
    dP.copy_(g)
    dS = torch.empty_strided(P.size(), P.stride(), device=DEV)
    ld = P.stride(-2)
    dT = ops.softmax_posbias_backward(dP, ld, Sraw, ld, lse, B * M * N, N, stat[2:], 500.0, p, seed, ld, dS, ld, table,
                                      (R, grid, w), True)
    s64 = Sraw.detach().cpu().double().requires_grad_()
    t64 = table.cpu().double().requires_grad_()
    Pr = torch.softmax(s64 + w * dense_bias(t64, R, grid), -1) * keep / (1 - p)
    torch.testing.assert_close(P.cpu().double(), Pr.detach(), rtol=2e-3, atol=2e-6)
    (Pr * g.cpu().double()).sum().backward()
    torch.testing.assert_close(dS.cpu().double(), s64.grad, rtol=5e-3, atol=1e-5)
    torch.testing.assert_close(dT.cpu().double(), t64.grad, rtol=1e-3, atol=1e-4)


def test_cuda_graph_replay_with_dropout_is_reproducible():
    grid = (5, 6, 7)
    enc = _bias_encoder(grid, [32, 32, 32], dropout=0.1).train()
    N = math.prod(grid)
    x = torch.randn(2, N, 32, device=DEV, requires_grad=True)
    pos, vm = torch.ones(2, N, 3, device=DEV), torch.ones(2, N, 1, device=DEV)
    tbl = enc.pos_code_layer.pos_coder.biases

    def step():
        tbl.grad = None
        x.grad = None
        y = enc(x, pos, vm, torch.Size(grid))
        y.sum().backward()
        return y, tbl.grad

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y_g, dT_g = step()
    runs = []
    for base in (1234, 1234, 99):
        ops.reseed(base)
        g.replay()
        torch.cuda.synchronize()
        runs.append((y_g.detach().clone(), dT_g.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert not torch.equal(runs[0][0], runs[2][0])          # a new base seed draws new masks
    assert float(runs[0][1].abs().max()) > 0
