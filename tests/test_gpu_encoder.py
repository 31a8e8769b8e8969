"""GPU parity of the CUDA SegtranFusionEncoder against the golden fixtures produced by the real reference
(and, transitively, the oracle).  Tolerance: 1e-3 rel on outputs (BASELINE.json north_star), written below."""
import pytest
import torch

from tests.helpers import build_b200_encoder, load_golden, rel_err, rms_rel

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-3          # max|a-b| / max|b|, forward outputs (north_star tolerance)
GRAD_TOL = 5e-3         # gradients: same arithmetic (TF32 operands, fp32 accumulation) through ~2x as many GEMMs
CASES = ["enc3d_small", "enc2d_compress", "enc3d_ragged", "enc2d_nosqueeze", "enc3d_sqffn", "enc3d_sharedout"]   # --nosqueeze, --squeezeuseffn, trans_output_type=shared


def _run(name, need_grad):
    fx = load_golden(name)
    enc = build_b200_encoder(fx).eval()
    x = fx["x"].cuda().requires_grad_(need_grad)
    pos = fx["voxels_pos"].cuda()
    y = enc(x, pos, fx["vmask"].cuda(), torch.Size(fx["grid"]))
    return fx, enc, x, y


@pytest.mark.parametrize("name", CASES)
def test_forward_matches_reference(name):
    with torch.no_grad():
        fx, enc, x, y = _run(name, False)
    assert y.shape == fx["out"].shape
    e = rel_err(y, fx["out"])
    print(name, "fwd rel", e, "rms", rms_rel(y, fx["out"]))
    assert e < OUT_TOL


@pytest.mark.parametrize("name", CASES)
def test_backward_matches_reference(name):
    fx, enc, x, y = _run(name, True)
    (y * fx["G"].cuda()).sum().backward()
    e = rel_err(x.grad, fx["grad_x"])
    print(name, "dx rel", e)
    assert e < GRAD_TOL
    gscale = max(float(g.abs().max()) for g in fx["grad_params"].values())
    got = dict(enc.named_parameters())
    for k, g in fx["grad_params"].items():
        gg = got[k].grad
        if float(g.abs().max()) == 0.0:          # never-used / shift-invariant parameters
            assert gg is None or float(gg.abs().max()) <= 1e-5 * gscale, k
            continue
        assert gg is not None, k
        err = float((gg.cpu() - g).abs().max())
        assert err <= GRAD_TOL * float(g.abs().max()) + 2e-5 * gscale, (k, err, float(g.abs().max()))


@pytest.mark.parametrize("name", CASES)
def test_tf32x3_mode_matches_reference_to_fp32_level(name):
    """Validation mode (ops.set_precision('tf32x3')): no producer rounds to TF32 and every GEMM runs as three passes on
    the hi/lo operand splits.  Forward and gradients then agree with the reference to fp32 round-off, which shows that
    the kernels, the fused epilogues and the re-associated algebra are exact and that TF32 operand rounding is the
    only deviation of the default mode."""
    from segtran_b200 import ops
    ops.set_precision("tf32x3")
    try:
        fx, enc, x, y = _run(name, True)
        e = rel_err(y, fx["out"])
        (y * fx["G"].cuda()).sum().backward()
        ex = rel_err(x.grad, fx["grad_x"])
        print(name, "tf32x3 fwd rel %.2e dx rel %.2e" % (e, ex))
        assert e < 2e-5 and ex < 1e-4
        gscale = max(float(g.abs().max()) for g in fx["grad_params"].values())
        got = dict(enc.named_parameters())
        for k, g in fx["grad_params"].items():
            if float(g.abs().max()) == 0.0:
                continue
            err = float((got[k].grad.cpu() - g).abs().max())
            assert err <= 1e-4 * float(g.abs().max()) + 1e-6 * gscale, (k, err, float(g.abs().max()))
    finally:
        ops.set_precision("tf32")


def test_clamp_case_matches_reference():
    """Scores beyond attn_clip=500 (segtran_shared.py:578-580): squeeze-out max is ~6000 -> clamped, in-squeeze
    (max 477) is not.  Softmax over saturated scores amplifies operand rounding, hence the looser bound."""
    with torch.no_grad():
        fx, enc, x, y = _run("enc3d_clamp", False)
    t = enc.translayers[0]
    assert t.ator_out_trans.clamp_count == 1 and t.in_ator_trans.clamp_count == 0
    assert abs(t.ator_out_trans.max_attn - fx["max_attn"][1]) < 1e-2 * fx["max_attn"][1]
    assert rel_err(y, fx["out"]) < 5e-2
    from segtran_b200 import ops
    ops.set_precision("tf32x3")          # with fp32-level products the saturated softmax agrees tightly too
    try:
        with torch.no_grad():
            fx, enc, x, y = _run("enc3d_clamp", False)
        print("clamp tf32x3 rel", rel_err(y, fx["out"]))
        assert rel_err(y, fx["out"]) < 1e-3
    finally:
        ops.set_precision("tf32")


def test_training_mode_dropout_runs_and_is_consistent():
    """Dropout on (reference default 0.2): finite outputs/gradients, masks change from step to step (device-side
    seed advance), and the whole step replays under a CUDA graph with a fresh mask per replay."""
    from segtran_b200 import ops
    from segtran_b200.graph import CapturedStep
    fx = load_golden("enc3d_small")
    enc = build_b200_encoder(fx, dropout=0.2).train()
    x = fx["x"].cuda().requires_grad_()
    pos, mask, grid = fx["voxels_pos"].cuda(), fx["vmask"].cuda(), torch.Size(fx["grid"])
    y1 = enc(x, pos, mask, grid)
    y2 = enc(x, pos, mask, grid)
    assert torch.isfinite(y1).all() and not torch.equal(y1, y2)
    y1.square().mean().backward()
    assert torch.isfinite(x.grad).all()
    # expectation over masks stays close to the no-dropout output (inverted dropout keeps the mean)
    enc.eval()
    with torch.no_grad():
        y0 = enc(x, pos, mask, grid)
    enc.train()
    acc = torch.zeros_like(y0)
    with torch.no_grad():
        for _ in range(64):
            acc += enc(x, pos, mask, grid)
    assert rel_err(acc / 64, y0) < 0.25

    # graph capture: fresh module and input that have never been used on the (legacy) default stream — autograd binds
    # a leaf's gradient accumulation to the stream of its first use, and that must not be the legacy stream
    enc2 = build_b200_encoder(fx, dropout=0.2).train()
    x2 = fx["x"].cuda().requires_grad_()

    def step():
        x2.grad = None
        for p_ in enc2.parameters():
            p_.grad = None
        out = enc2(x2, pos, mask, grid)
        out.square().mean().backward()
        return out

    g = CapturedStep(step, warmup=2)
    a = g().clone()
    b = g().clone()
    assert torch.isfinite(a).all() and not torch.equal(a, b)       # new mask on every replay
    assert g.kernel_launches > 20


def test_direct_gradient_accumulation_equals_autograd():
    """GradBucket(direct_accumulate=True): weight-gradient GEMMs / column sums add straight into the flat bucket (autograd
    gets None for those inputs).  Same gradients as the stock AccumulateGrad path, twice in a row (accumulation)."""
    from segtran_b200 import ops
    from segtran_b200.parallel import GradBucket
    fx = load_golden("enc3d_small")
    enc = build_b200_encoder(fx).eval()
    x = fx["x"].cuda()
    pos, mask, G = fx["voxels_pos"].cuda(), fx["vmask"].cuda(), fx["G"].cuda()

    def run():
        y = enc(x, pos, mask, torch.Size(fx["grid"]))
        (y * G).sum().backward()

    run()
    want = {k: p.grad.clone() for k, p in enc.named_parameters() if p.grad is not None}
    for p in enc.parameters():
        p.grad = None
    try:
        bucket = GradBucket(enc.parameters(), direct_accumulate=True)
        run()
        run()                                   # second pass accumulates on top of the first
        for k, p in enc.named_parameters():
            if k in want:
                ref = 2.0 * want[k]
                assert float((p.grad - ref).abs().max()) <= 1e-5 * float(ref.abs().max()) + 1e-9, k
        bucket.zero()
        assert all(float(p.grad.abs().max()) == 0.0 for p in enc.parameters())
    finally:
        ops.set_grad_sink(False)
