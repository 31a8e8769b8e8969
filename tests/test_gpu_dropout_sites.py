"""Per-site evidence for the regenerated (counter-based) dropout masks: every dropout site of the hot path
(segtran_shared.py:944 feature dropout in the prologue, :605 attention dropout, :245 MMSharedMid, :273 MMPrivateOutput) keeps
elements at rate 1-p, scales the kept ones by 1/(1-p), is deterministic in its seed, differs between seeds, shows no row /
column structure, and the backward pass applies the SAME mask as the forward pass (the masks are never stored).
The attention site of the fused wgmma kernel is covered in test_gpu_attn.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu
P = 0.3


@pytest.fixture(autouse=True)
def _fp32_grade_precision():
    """tf32x3 mode: no kernel rounds its output to TF32 for a following tensor-core operand, so kept values can be compared
    with (no-dropout value) / (1-p) to fp32 accuracy.  The masks do not depend on the precision mode."""
    from segtran_b200 import ops
    ops.set_precision("tf32x3")
    yield
    ops.set_precision("tf32")


def _check_mask(kept, p=P, row_tol=0.1, col_tol=0.1):
    rate = float(kept.float().mean())
    n = kept.numel()
    assert abs(rate - (1 - p)) < 5 * (p * (1 - p) / n) ** 0.5 + 1e-4, rate           # 5 sigma of the binomial
    k2 = kept.reshape(-1, kept.shape[-1]).float()
    assert float((k2.mean(1) - (1 - p)).abs().max()) < row_tol                          # no dead / always-kept rows
    assert float((k2.mean(0) - (1 - p)).abs().max()) < col_tol                          # ... or columns
    # neighbouring elements are uncorrelated (the hash words cover groups of 4 consecutive elements)
    a, b = k2[:, :-1] - (1 - p), k2[:, 1:] - (1 - p)
    corr = float((a * b).mean() / (p * (1 - p)))
    assert abs(corr) < 0.01, corr


def test_prologue_feature_dropout_mask():
    from segtran_b200 import ops
    torch.manual_seed(0)
    B, N, C = 2, 1000, 1024
    x = torch.randn(B, N, C, device="cuda", requires_grad=True)
    g, b = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
    pe = torch.randn(N, C, device="cuda")
    mask = torch.ones(B, N, 1, device="cuda")
    h0 = ops.prologue(x, g, b, pe, 1.0, mask, 0.0, 0)
    ha = ops.prologue(x, g, b, pe, 1.0, mask, P, 77)
    hb = ops.prologue(x, g, b, pe, 1.0, mask, P, 77)
    hc = ops.prologue(x, g, b, pe, 1.0, mask, P, 78)
    assert torch.equal(ha, hb) and not torch.equal(ha, hc)
    kept = ha != 0
    _check_mask(kept)
    assert torch.allclose(ha[kept], (h0 / (1 - P))[kept], rtol=1e-5, atol=1e-6)
    # masks of two seeds are independent: P(kept in both) = (1-p)^2
    both = float(((ha != 0) & (hc != 0)).float().mean())
    assert abs(both - (1 - P) ** 2) < 3e-3, both


def test_softmax_attention_dropout_mask_and_backward_uses_it():
    from segtran_b200 import ops
    torch.manual_seed(1)
    S = torch.randn(2, 4, 300, 512, device="cuda", requires_grad=True)
    P0 = ops.softmax(S.detach(), None, 500.0, 0.0, 0)
    Pa = ops.softmax(S, None, 500.0, P, 5)
    Pb = ops.softmax(S.detach(), None, 500.0, P, 5)
    assert torch.equal(Pa.detach(), Pb)
    kept = Pa.detach() != 0
    _check_mask(kept)
    assert torch.allclose(Pa.detach()[kept], (P0 / (1 - P))[kept], rtol=1e-5, atol=0)
    # backward with the regenerated mask: d/dS sum(G * dropout(softmax(S))) = softmax-backward of (G * mask / (1-p))
    G = torch.randn_like(P0)
    (Pa * G).sum().backward()
    Sr = S.detach().clone().requires_grad_()
    (torch.softmax(Sr, -1) * (G * kept / (1 - P))).sum().backward()
    assert float((S.grad - Sr.grad).abs().max()) < 1e-5 * max(1.0, float(Sr.grad.abs().max()))


def test_gemm_epilogue_dropout_mask_mid_layer():
    """MMSharedMid: dropout(gelu(x W^T + b)) in the epilogue of the wgmma GEMM, mask regenerated in the backward epilogue."""
    from segtran_b200 import ops
    torch.manual_seed(2)
    x = torch.randn(2, 640, 512, device="cuda", requires_grad=True)
    W = (torch.randn(768, 512, device="cuda") * 0.05).requires_grad_()
    b = (torch.randn(768, device="cuda") * 0.1).requires_grad_()
    y0 = ops.linear(x.detach(), W.detach(), b.detach(), gelu=True, round_out=False)
    ya = ops.linear(x, W, b, gelu=True, drop_p=P, seed=11, round_out=False)
    yb = ops.linear(x.detach(), W.detach(), b.detach(), gelu=True, drop_p=P, seed=11, round_out=False)
    yc = ops.linear(x.detach(), W.detach(), b.detach(), gelu=True, drop_p=P, seed=12, round_out=False)
    assert torch.equal(ya.detach(), yb) and not torch.equal(yb, yc)
    kept = yb != 0
    _check_mask(kept)
    assert torch.allclose(yb[kept], (y0 / (1 - P))[kept], rtol=1e-5, atol=1e-7)
    # backward: the bias gradient is the column sum of G * mask * gelu'(h) / (1-p): exactly zero contribution where dropped
    G = torch.ones_like(y0)
    ya.backward(G)
    h = torch.nn.functional.linear(x.detach(), W.detach(), b.detach())
    gp = 0.5 * (1 + torch.erf(h / 2 ** 0.5)) + h * torch.exp(-0.5 * h * h) / (2 * torch.pi) ** 0.5
    ref = (gp * kept / (1 - P)).sum((0, 1))
    assert float((b.grad - ref).abs().max()) < 2e-3 * float(ref.abs().max())


def test_ln_softaggr_input_dropout_mask_seen_through_the_gradient():
    """MMPrivateOutput: LN(dropout(Y)) — dropped inputs cannot be seen in the output, but dY is exactly zero there."""
    from segtran_b200 import ops
    torch.manual_seed(3)
    B, M, N, F = 2, 4, 500, 1024
    Y = torch.randn(B, M, N, F, device="cuda", requires_grad=True)
    g = torch.ones(F, device="cuda", requires_grad=True)
    b = torch.zeros(F, device="cuda", requires_grad=True)
    ws = (torch.randn(1, F, device="cuda") * 0.02).requires_grad_()
    bs = torch.zeros(1, device="cuda", requires_grad=True)
    out = ops.ln_softaggr(Y, g, b, ws, bs, P, 21)
    out2 = ops.ln_softaggr(Y.detach(), g.detach(), b.detach(), ws.detach(), bs.detach(), P, 21)
    assert torch.equal(out.detach(), out2)
    out.backward(torch.randn_like(out))
    kept = Y.grad != 0
    _check_mask(kept)
    # the forward used the same mask: recompute with an explicit mask in PyTorch
    Yd = Y.detach() * kept / (1 - P)
    Yn = torch.nn.functional.layer_norm(Yd, (F,), g.detach(), b.detach(), 1e-12)
    w = torch.softmax(Yn @ ws.detach().t() + bs.detach(), dim=1)
    ref = (Yn * w).sum(1)
    assert float((out.detach() - ref).abs().max()) < 1e-4 * float(ref.abs().max())
