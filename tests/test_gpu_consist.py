"""The attention-consistency loss kernels (csrc/sx_consist.cu) on the GPU: the drop-in losses against the reference's
fixtures (oracle/gen_consist_golden.py), the cfg-4 shape against the float64 oracle, dense against pair input,
run-to-run bit identity, CUDA-graph replay, no [B,N,N] allocation in a forward that needs no gradient, and
SegtranFusionEncoder with --attnconsist plus the loss against encoder-driven reference fixtures (clamped scores included)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from segtran_b200 import ops, train  # noqa: E402
from oracle import consist_oracle as CO  # noqa: E402
import segtran_b200.networks.segtran_shared as S  # noqa: E402
from tests.helpers import encoder_config  # noqa: E402

DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def _entries(fx, dev=DEV, dtype=torch.float32):
    return [[t.to(dev, dtype).clone().requires_grad_() for t in e] if isinstance(e, list) else
            e.to(dev, dtype).clone().requires_grad_() for e in fx["entries"]]


def _flat(entries):
    return [t for e in entries for t in (e if isinstance(e, list) else [e])]


def _run(fx, entries):
    fun = train.attn_consist_loss3d if fx["three_d"] else train.attn_consist_loss2d
    kw = {} if fx["only_first_layer"] is None else {"only_first_layer": fx["only_first_layer"]}
    return fun(entries, torch.Size(fx["grid"]), fx["mask"].to(DEV), **kw)


def _maxrel(got, ref):
    ref = ref.to(got.device, torch.float64)
    return float((got.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


@pytest.fixture
def precision():
    old = ops.get_precision()
    yield ops.set_precision
    ops.set_precision(old)


# 2-D pair fixtures are checked in tf32x3 only: a TF32 product can move an element across the mu / mu - 0.1 thresholds
# (the margin rule at TF32 is checked on threshold-safe inputs in test_margin_tf32_against_float64_oracle)
CASES = [("consist3d_pair", "tf32"), ("consist3d_pair", "tf32x3"), ("consist3d_pair2", "tf32"),
         ("consist3d_pair2", "tf32x3"), ("consist2d_pair", "tf32x3"), ("consist2d_pair_cap", "tf32x3"),
         ("consist2d_dense", "tf32"), ("consist3d_dense", "tf32")]


@pytest.mark.parametrize("name,prec", CASES)
def test_loss_matches_reference_fixture(name, prec, precision):
    precision(prec)
    fx = _load(name)
    ent = _entries(fx)
    loss = _run(fx, ent)
    assert loss.dim() == 0
    loss.backward()
    fwd_tol, grad_tol = (1e-3, 5e-3) if prec == "tf32" else (2e-5, 1e-4)
    assert abs(float(loss) - float(fx["loss"])) <= fwd_tol * max(1.0, abs(float(fx["loss"])))
    for t, g in zip(_flat(ent), fx["grads"]):
        got = torch.zeros_like(t) if t.grad is None else t.grad
        if float(g.abs().max()) == 0.0:
            assert float(got.abs().max()) == 0.0
        else:
            assert _maxrel(got, g) <= grad_tol, name


def _cfg4(seed=0, B=4, N=2744, A=1024, K=4):
    g = torch.Generator(device=DEV).manual_seed(seed)
    xi = (torch.randn(B, 1, A, N, device=DEV, generator=g) * 0.05).requires_grad_()
    xo = (torch.randn(B, 1, N, A, device=DEV, generator=g) * 0.05).requires_grad_()
    lab = torch.randint(0, K, (B, 28, 28, 28), device=DEV, generator=g)
    mask = torch.nn.functional.one_hot(lab, K).permute(0, 4, 1, 2, 3).float()
    return [[xi, xo]], mask


def test_cfg4_bce_against_float64_oracle():
    ent, mask = _cfg4()
    loss = train.attn_consist_loss3d(ent, (14, 14, 14), mask)
    loss.backward()
    ref_ent = [[t.detach().double().requires_grad_() for t in ent[0]]]
    ref = CO.consist_loss3d(ref_ent, (14, 14, 14), mask.double())
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-3 * abs(float(ref))
    for t, r in zip(ent[0], ref_ent[0]):
        assert _maxrel(t.grad, r.grad) <= 5e-3


def test_dense_matches_pair_on_the_same_affinity(precision):
    precision("tf32x3")
    g = torch.Generator(device=DEV).manual_seed(3)
    B, N, A, K = 2, 300, 64, 3
    xi = torch.randn(B, 1, A, N, device=DEV, generator=g) * 0.2
    xo = torch.randn(B, 1, N, A, device=DEV, generator=g) * 0.2
    x = torch.matmul(xo.double(), xi.double()).float()
    lab = torch.randint(0, K, (B, 30, 20), device=DEV, generator=g)
    mask = torch.nn.functional.one_hot(lab, K).permute(0, 3, 1, 2).float()
    a = [xi.clone().requires_grad_(), xo.clone().requires_grad_()]
    d = x.clone().requires_grad_()
    # margin variant: an element within rounding of a threshold may flip; its effect on the loss is far below 1e-4
    la = train.attn_consist_loss2d([a], (15, 20), mask)
    ld = train.attn_consist_loss2d([d], (15, 20), mask)
    assert abs(float(la) - float(ld)) <= 1e-4 * max(1.0, abs(float(ld)))
    la3 = train.attn_consist_loss3d([a], (1, 15, 20), mask.unsqueeze(-1))     # [B,K,H,W,D=1]
    ld3 = train.attn_consist_loss3d([d], (1, 15, 20), mask.unsqueeze(-1))
    assert abs(float(la3) - float(ld3)) <= 1e-5 * abs(float(ld3))
    (la3 + ld3).backward()
    # d loss / d X (dense) against the chain rule through the pair's gradients: dXo = dX Xi^T
    dxo = torch.matmul(d.grad.double(), xi.double().transpose(-1, -2))
    assert _maxrel(a[1].grad, dxo) <= 1e-4


def test_bit_identical_across_runs():
    outs = []
    for _ in range(2):
        ent, mask = _cfg4(seed=5, N=1000, A=256)
        loss = train.attn_consist_loss3d(ent, (10, 10, 10), mask[:, :, :20, :20, :20])
        loss.backward()
        fx = _load("consist2d_pair_cap")
        e2 = _entries(fx)
        l2 = _run(fx, e2)
        l2.backward()
        outs.append([loss.detach().clone(), ent[0][0].grad, ent[0][1].grad, l2.detach().clone()] +
                    [t.grad for t in _flat(e2)])
    for u, v in zip(*outs):
        assert torch.equal(u, v)


def test_cuda_graph_replay_with_the_2d_cap():
    fx = _load("consist2d_pair_cap")
    ent = _entries(fx)
    mask = fx["mask"].to(DEV)
    grads = [torch.zeros_like(t) for t in _flat(ent)]

    def step():
        loss = train.attn_consist_loss2d(ent, torch.Size(fx["grid"]), mask)
        gs = torch.autograd.grad(loss, _flat(ent))
        for b, gg in zip(grads, gs):
            b.copy_(gg)
        return loss

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager = step().detach().clone()
    torch.cuda.current_stream().wait_stream(s)
    eager_grads = [b.clone() for b in grads]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for b in grads:
        b.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert float(out) == float(eager) == 1.0
    for b, e in zip(grads, eager_grads):
        assert torch.equal(b, e)
    # new inputs, same graph: the cap factor is recomputed on the device
    with torch.no_grad():
        for t in _flat(ent):
            t.mul_(0.01)
    graph.replay()
    ref_ent = [[t.detach().double().cpu().requires_grad_() for t in e] for e in ent]
    ref = CO.consist_loss2d(ref_ent, torch.Size(fx["grid"]), fx["mask"].double())
    assert float(ref) < 1.0 and abs(float(out) - float(ref)) <= 1e-3 * abs(float(ref))


def test_forward_without_grad_allocates_no_affinity_matrix():
    B, N, A = 4, 2744, 1024
    ent, mask = _cfg4()
    ent = [[t.detach() for t in ent[0]]]
    train.attn_consist_loss3d(ent, (14, 14, 14), mask)       # warm-up: scratch buffers
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    loss = train.attn_consist_loss3d(ent, (14, 14, 14), mask)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < B * N * N * 4     # the packed operands only (2 x B*N*A)
    assert torch.isfinite(loss)


# ---------------------------------------------------------------------------------------------------------------------
# the margin variant at the default TF32 precision, on inputs whose affinities are exact in TF32 and keep away from the
# mu / mu - 0.1 thresholds (entries in {-1, 0, 1} / 8: every X is a multiple of 1/64, every product and sum exact)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,A", [(2, 15, 20, 64), (4, 49, 56, 1024)])
def test_margin_tf32_against_float64_oracle(B, H, W, A):
    N, K = H * W, 4
    g = torch.Generator().manual_seed(0)
    xi = (torch.randint(-1, 2, (B, 1, A, N), generator=g).float() * 0.125).to(DEV).requires_grad_()
    xo = (torch.randint(-1, 2, (B, 1, N, A), generator=g).float() * 0.125).to(DEV).requires_grad_()
    lab = torch.randint(0, K, (B, 2 * H, 2 * W), generator=g)
    mask = torch.nn.functional.one_hot(lab, K).permute(0, 3, 1, 2).float().to(DEV)
    ref_ent = [[xi.detach().double().requires_grad_(), xo.detach().double().requires_grad_()]]
    x = torch.matmul(ref_ent[0][1], ref_ent[0][0]).squeeze(1).detach()
    mu = x.mean(dim=(1, 2))
    q = 1.0 / 64
    for v in (mu, mu - 0.1):                    # the precondition that makes the classification exact
        assert float(((v / q) - torch.round(v / q)).abs().min() * q) > 1e-6
    loss = train.attn_consist_loss2d([[xi, xo]], (H, W), mask)
    loss.backward()
    ref = CO.consist_loss2d(ref_ent, (H, W), mask.double())
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-3 * abs(float(ref))
    for t, r in zip((xi, xo), ref_ent[0]):
        assert _maxrel(t.grad, r.grad) <= 5e-3


# ---------------------------------------------------------------------------------------------------------------------
# SegtranFusionEncoder (--attnconsist) + the loss against the reference encoder and loss
# ---------------------------------------------------------------------------------------------------------------------
ENC_CASES = [("consist_enc3d", "tf32"), ("consist_enc3d", "tf32x3"), ("consist_enc3d_2l", "tf32"),
             ("consist_enc3d_2l", "tf32x3"), ("consist_enc2d", "tf32x3"), ("consist_enc2d_cap", "tf32x3"),
             ("consist_enc2d_dense", "tf32x3"), ("consist_enc3d_dense", "tf32"),
             ("consist_enc3d_dense", "tf32x3"), ("consist_enc_clamp", "tf32x3")]


def _consist_encoder(fx):
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"], num_attractors=fx["num_attractors"],
                         pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"])
    cfg.use_squeezed_transformer = fx["use_squeezed_transformer"]
    cfg.use_attn_consist_loss = True
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    enc.apply(S.SegtranInitWeights(cfg).tie_qk)
    enc.load_state_dict(fx["state_dict"], strict=True)
    return enc.to(DEV).eval()


@pytest.mark.parametrize("name,prec", ENC_CASES)
def test_encoder_plus_loss_matches_reference_fixture(name, prec, precision):
    precision(prec)
    fx = _load(name)
    enc = _consist_encoder(fx)
    x = fx["x"].to(DEV).requires_grad_()
    enc(x, fx["voxels_pos"].to(DEV), fx["vmask"].to(DEV), torch.Size(fx["grid"]))
    fun = train.attn_consist_loss3d if fx["three_d"] else train.attn_consist_loss2d
    kw = {} if fx["only_first_layer"] is None else {"only_first_layer": fx["only_first_layer"]}
    loss = fun(enc.layers_attn_scores, torch.Size(fx["grid"]), fx["mask"].to(DEV), **kw)
    loss.backward()
    fwd_tol, grad_tol = (1e-3, 5e-3) if prec == "tf32" else (2e-5, 2e-4)
    ref = float(fx["loss"])
    assert abs(float(loss) - ref) <= fwd_tol * max(1.0, abs(ref)), (float(loss), ref)
    params = dict(enc.named_parameters())
    gscale = max(float(g.abs().max()) for g in fx["grad_params"].values())
    checked = set()
    # the margin rule is invariant under X -> X + const (mu moves with X), so with dense entries the gradient of
    # attn_scaler.bias is zero in exact arithmetic: both sides hold rounding noise, bounded against the gradient scale
    shift_invariant = {"attn_scaler.bias"} if not fx["three_d"] and not fx["use_squeezed_transformer"] else set()
    for k, gref in fx["grad_params"].items():
        ours = params[k].grad
        if k in shift_invariant:
            assert float(gref.abs().max()) <= 1e-3 * gscale and float(ours.abs().max()) <= 1e-3 * gscale, k
            continue
        if float(gref.abs().max()) == 0.0:
            assert ours is None or float(ours.abs().max()) <= 1e-5 * gscale, k
            continue
        assert ours is not None, k
        err = float((ours.cpu() - gref).abs().max()) / (float(gref.abs().max()) + 4e-3 * gscale)
        assert err <= grad_tol, (k, err)
        checked.add(k.split(".")[0])
    assert "attn_scaler" in checked and "translayers" in checked
    assert _maxrel(x.grad, fx["grad_x"]) <= grad_tol
    if name == "consist_enc_clamp":                # the squeeze-out scores were clamped (max_attn ~2100 > 500)
        assert enc.translayers[0].ator_out_trans.clamp_count == 1
