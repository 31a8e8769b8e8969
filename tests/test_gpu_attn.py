"""Fused attention kernels (csrc/sx_attn.cu and the softmax-backward epilogue of sx_gemm) against plain fp32 PyTorch
of the same operation (reference segtran_shared.py:566-567, :569-580, :601, :605)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _tf32(x):
    """round to the nearest TF32 value (what the producers of q/k do in the default precision)"""
    y = x.clone()
    y.view(torch.int32).add_(0x1000).bitwise_and_(-8192)
    return y


def _ref_probs(q, k, M, clip):
    Bq, U1, C = q.shape
    B, U2, _ = k.shape
    d = C // M
    qv = q.double().view(Bq, U1, M, d).permute(0, 2, 1, 3)
    kv = k.double().view(B, U2, M, d).permute(0, 2, 1, 3)
    s = qv @ kv.transpose(-1, -2) / math.sqrt(d)
    if float(s.max()) > clip:
        s = s.clamp(-clip, clip)
    return s, torch.softmax(s, dim=-1)


@pytest.mark.parametrize("B,Bq,M,U1,U2,d,scale", [
    (2, 2, 4, 300, 256, 64, 1.0),       # single pass (keys fit one accumulator), row tail
    (2, 1, 4, 700, 1024, 256, 1.0),     # cfg-4 widths: two passes over four key chunks, shared queries
    (1, 1, 1, 105, 77, 12, 1.0),        # ragged everything, K tail, one mode
    (2, 2, 2, 513, 300, 36, 1.0),       # ragged key count across two chunks
    (1, 1, 4, 260, 512, 32, 40.0),      # scores beyond the clamp
])
def test_attn_probs_fused_matches_torch(B, Bq, M, U1, U2, d, scale):
    from segtran_b200 import ops
    torch.manual_seed(U1 + U2)
    q = _tf32(torch.randn(Bq, U1, M * d, device="cuda") * scale)
    k = _tf32(torch.randn(B, U2, M * d, device="cuda") * scale)
    diag = torch.tensor([-3.0e38, 0.0, 0.0], device="cuda")
    P, S, lse, rowmax, stat = ops.attn_probs_fused(q, k, M, clip=500.0, diag=diag, need_scores=True, round_out=False)
    torch.cuda.synchronize()
    s_ref, p_ref = _ref_probs(q, k, M, 500.0)
    s_raw = (q.double().view(Bq, U1, M, d).permute(0, 2, 1, 3) @
             k.double().view(B, U2, M, d).permute(0, 2, 1, 3).transpose(-1, -2)) / math.sqrt(d)
    assert (S.double() - s_raw).abs().max() <= 2e-6 * s_raw.abs().max()
    tol = 5e-5 if scale > 1 else 2e-6           # saturated rows amplify the last-bit differences of the scores
    assert (P.double() - p_ref).abs().max() < tol
    assert (P.sum(-1) - 1).abs().max() < 1e-5
    lse_ref = torch.logsumexp(s_ref, dim=-1)
    assert (lse.double() - lse_ref).abs().max() <= 1e-5 * lse_ref.abs().max().clamp_min(1.0)
    assert (rowmax.double() - s_raw.max(-1).values).abs().max() <= 2e-6 * s_raw.abs().max()
    mx, cnt, amb = diag.tolist()
    assert abs(mx - float(s_raw.max())) <= 2e-6 * float(s_raw.abs().max())
    assert cnt == (1.0 if float(s_raw.max()) > 500.0 else 0.0) and amb == 0.0


def test_attn_probs_fused_dropout_statistics_and_determinism():
    from segtran_b200 import ops
    torch.manual_seed(3)
    B, M, U1, U2, d = 2, 4, 384, 1024, 64
    q = _tf32(torch.randn(B, U1, M * d, device="cuda"))
    k = _tf32(torch.randn(B, U2, M * d, device="cuda"))
    P0 = ops.attn_probs_fused(q, k, M, round_out=False)[0]
    Pa = ops.attn_probs_fused(q, k, M, drop_p=0.2, seed=1234, round_out=False)[0]
    Pb = ops.attn_probs_fused(q, k, M, drop_p=0.2, seed=1234, round_out=False)[0]
    Pc = ops.attn_probs_fused(q, k, M, drop_p=0.2, seed=99, round_out=False)[0]
    assert torch.equal(Pa, Pb) and not torch.equal(Pa, Pc)
    kept = Pa != 0
    rate = float(kept.float().mean())
    assert abs(rate - 0.8) < 2e-3, rate
    assert torch.allclose(Pa[kept], (P0 / 0.8)[kept], rtol=1e-6, atol=0)
    # independence across rows / columns: keep rates per row and per column stay binomial
    assert float((kept.float().mean(-1) - 0.8).abs().max()) < 0.08
    assert float((kept.float().mean(-2) - 0.8).abs().max()) < 0.12


def _sq_inputs(B, M, U1, U2, d, Fd, seed=0, bq=None):
    torch.manual_seed(seed)
    bq = B if bq is None else bq
    dev = "cuda"
    q = _tf32(torch.randn(bq, U1, M * d, device=dev)).requires_grad_()
    k = _tf32(torch.randn(B, U2, M * d, device=dev)).requires_grad_()
    vp = _tf32(torch.randn(B, U2, M * Fd, device=dev) * 0.5).requires_grad_()
    bm = (torch.randn(Fd, device=dev) * 0.1).requires_grad_()
    Wo = torch.nn.Parameter(torch.randn(M * Fd, Fd, 1, device=dev) * 0.05)
    bo = torch.nn.Parameter(torch.randn(M * Fd, device=dev) * 0.1)
    gY = torch.randn(B, M, U1, Fd, device=dev)
    return q, k, vp, bm, Wo, bo, gY


def _fused(q, k, vp, M, att_p, s1, bm, hid_p, s2, Wo, bo, diag):
    """The fused squeeze-out of CrossAttFeatTrans + ExpandedFeatTrans: dQ reads a K-major copy of the keys."""
    from segtran_b200 import ops
    P = ops.attn_probs(q, k, M, None, 500.0, att_p, s1, diag, kmajor_dq=True)
    return ops.attn_pv_gelu_group_linear(P, vp, M, bm, hid_p, s2, Wo, bo)


def _unfused(q, k, vp, M, att_p, s1, bm, hid_p, s2, Wo, bo):
    from segtran_b200 import ops
    amax = torch.full((1,), -3.0e38, device=q.device)
    s = ops.attn_scores(q, k, M, amax)
    P = ops.softmax(s, amax, 500.0, att_p, s1, None)
    return ops.attn_pv_gelu_group_linear(P, vp, M, bm, hid_p, s2, Wo, bo)


@pytest.mark.parametrize("B,bq,M,U1,U2,d,Fd,att_p,hid_p", [
    (2, 2, 4, 300, 256, 32, 64, 0.0, 0.0),
    (2, 1, 4, 520, 1024, 64, 128, 0.0, 0.0),          # two-pass scores, shared queries (dq reduced over the batch)
    (2, 2, 2, 260, 300, 32, 64, 0.2, 0.2),            # both dropouts: masks regenerated in the fused backward
])
def test_fused_squeeze_out_matches_unfused_path(B, bq, M, U1, U2, d, Fd, att_p, hid_p):
    """Same seeds -> same dropout masks: the fused node (sx_attn + softmax-backward GEMM epilogue) must reproduce the
    separate-kernel path (attn_scores -> sx_softmax -> P.V GEMM -> sx_softmax_bwd) in outputs and all gradients."""
    outs = []
    for fused in (True, False):
        q, k, vp, bm, Wo, bo, gY = _sq_inputs(B, M, U1, U2, d, Fd, seed=5, bq=bq)
        diag = torch.tensor([-3.0e38, 0.0, 0.0], device="cuda")
        if fused:
            Y = _fused(q, k, vp, M, att_p, 1111, bm, hid_p, 2222, Wo, bo, diag)
        else:
            Y = _unfused(q, k, vp, M, att_p, 1111, bm, hid_p, 2222, Wo, bo)
        (Y * gY).sum().backward()
        outs.append([Y.detach()] + [t.grad.detach() for t in (q, k, vp, bm, Wo, bo)])
    names = ["Y", "dq", "dk", "dvp", "dbm", "dWo", "dbo"]
    for n, a, b in zip(names, outs[0], outs[1]):
        err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
        print(n, "fused vs unfused rel %.2e" % err)
        assert err < (2e-3 if n in ("dq", "dk") else 5e-4), (n, err)


def test_fused_squeeze_out_gradients_match_fp64_autograd():
    B, M, U1, U2, d, Fd = 2, 2, 200, 320, 32, 64
    q, k, vp, bm, Wo, bo, gY = _sq_inputs(B, M, U1, U2, d, Fd, seed=9)
    diag = torch.tensor([-3.0e38, 0.0, 0.0], device="cuda")
    Y = _fused(q, k, vp, M, 0.0, 0, bm, 0.0, 0, Wo, bo, diag)
    (Y * gY).sum().backward()
    got = [Y.detach()] + [t.grad.detach().clone() for t in (q, k, vp, bm, Wo, bo)]
    # fp64 autograd of the same math
    qd, kd, vd, bd, Wd, od = [t.detach().double().requires_grad_() for t in (q, k, vp, bm, Wo, bo)]
    s = (qd.view(B, U1, M, d).permute(0, 2, 1, 3) @ kd.view(B, U2, M, d).permute(0, 2, 3, 1)) / math.sqrt(d)
    P = torch.softmax(s, -1)
    U = P @ vd.view(B, U2, M, Fd).permute(0, 2, 1, 3)
    G = torch.nn.functional.gelu(U + bd)
    Yr = torch.einsum("bmnf,mof->bmno", G, Wd.view(M, Fd, Fd)) + od.view(1, M, 1, Fd)
    (Yr * gY.double()).sum().backward()
    ref = [Yr.detach()] + [t.grad for t in (qd, kd, vd, bd, Wd, od)]
    for n, a, b in zip(["Y", "dq", "dk", "dvp", "dbm", "dWo", "dbo"], got, ref):
        err = float((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30))
        print(n, "rel %.2e" % err)
        assert err < 3e-3, (n, err)             # TF32 operands (10-bit mantissa) in every contraction
