"""Per-kernel GPU tests: each segtran_b200 op against the same op written in plain PyTorch fp32 (on the GPU)."""

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def tf32(x):
    """round-to-nearest TF32 (what the library feeds the tensor cores)."""
    u = x.contiguous().view(torch.int32)
    u = (u + 0x0FFF + ((u >> 13) & 1)) & ~0x1FFF
    return u.view(torch.float32)


def close(a, b, tol):
    err = float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
    assert err < tol, err


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = False          # the PyTorch side of every comparison is true fp32
    torch.backends.cuda.matmul.allow_tf32 = False


def test_gemm_nt_all_majors_and_batch():
    from segtran_b200 import ops
    a = tf32(torch.randn(2, 3, 152, 72, device="cuda"))       # MN-major views need 16-byte pitches: 152 % 4 == 0
    b = tf32(torch.randn(2, 3, 260, 72, device="cuda"))
    ref = a.double() @ b.double().transpose(-1, -2)
    close(ops.gemm_nt(a, b, round_out=False).double(), ref, 1e-5)
    am = a.transpose(-1, -2).contiguous().transpose(-1, -2)       # MN-major view of the same values
    bm = b.transpose(-1, -2).contiguous().transpose(-1, -2)
    close(ops.gemm_nt(am, bm, round_out=False).double(), ref, 1e-5)
    close(ops.gemm_nt(a, bm, round_out=False).double(), ref, 1e-5)
    # broadcast B over z1, reduce over z1
    close(ops.gemm_nt(a, b[:1], round_out=False).double(), a.double() @ b[:1].double().transpose(-1, -2), 1e-5)
    red = ops.gemm_nt(am, bm, reduce_z1=True, round_out=False)
    close(red[0].double(), ref.sum(0), 1e-5)


def test_gemm_nt_tf32x3_recovers_fp32_products():
    """The 3-pass validation mode (A_hi B_hi + A_lo B_hi + A_hi B_lo) on UN-rounded fp32 operands: ~1e-6 of the fp64
    product, for every operand majorness, with the fused epilogue (bias + GELU + preact) and the accumulate path."""
    from segtran_b200 import ops
    a = torch.randn(2, 3, 152, 264, device="cuda")
    b = torch.randn(2, 3, 260, 264, device="cuda")
    bias = torch.randn(260, device="cuda")
    ref = a.double() @ b.double().transpose(-1, -2)
    e1 = float((ops.gemm_nt(a, b, round_out=False).double() - ref).abs().max() / ref.abs().max())
    ops.set_precision("tf32x3")
    try:
        am = a.transpose(-1, -2).contiguous().transpose(-1, -2)
        bm = b.transpose(-1, -2).contiguous().transpose(-1, -2)
        for x, y in ((a, b), (am, bm), (a, bm), (am, b)):
            close(ops.gemm_nt(x, y).double(), ref, 2e-6)
        h = torch.empty(2, 3, 152, 260, device="cuda")
        g = ops.gemm_nt(a, b, bias=bias, gelu=True, preact=h)
        close(h.double(), ref + bias.double(), 2e-6)
        close(g.double(), torch.nn.functional.gelu(ref + bias.double()), 2e-6)
        red = ops.gemm_nt(am, bm, reduce_z1=True)
        close(red[0].double(), ref.sum(0), 2e-6)
        acc = torch.ones(2, 3, 152, 260, device="cuda")
        ops.gemm_nt(a, b, out=acc, accumulate=True, alpha=0.5)
        close(acc.double(), 1.0 + 0.5 * ref, 2e-6)
    finally:
        ops.set_precision("tf32")
    assert e1 > 1e-5          # the single-pass mode on un-rounded operands is visibly TF32


def test_gemm_kernel_variants_agree():
    """The persistent kernel with one tile per CTA and with a grid of a few CTAs that each walk many tiles (operand
    ring and barrier phases carried across tiles) compute the same contract: same results on ragged, batched,
    MN-major, fused-epilogue and split-K / batch-reduced problems."""
    import segtran_b200._lib as L
    from segtran_b200 import ops
    a = tf32(torch.randn(2, 3, 300, 200, device="cuda"))
    b = tf32(torch.randn(2, 3, 520, 200, device="cuda"))
    am = a.transpose(-1, -2).contiguous().transpose(-1, -2)
    bias = torch.randn(520, device="cuda")

    def run():
        h = torch.empty(2, 3, 300, 520, device="cuda")
        y = ops.gemm_nt(a, b, bias=bias, gelu=True, preact=h, drop_p=0.25, seed=99)
        red = ops.gemm_nt(am, b, reduce_z1=True, round_out=False)
        sk = ops.gemm_nt(am, b[:1, :1], split_k=3, accumulate=True, out=torch.ones(2, 3, 300, 520, device="cuda"),
                         round_out=False)
        return y, h, red, sk

    try:
        ref = run()
        for ctas in (7, 1):
            L.call("sx_gemm_debug_set", b"max_ctas", ctas)
            got = run()
            assert torch.equal(got[0] == 0, ref[0] == 0)                  # identical dropout masks
            for g, r in zip(got, ref):
                close(g.double(), r.double(), 2e-6)
    finally:
        L.call("sx_gemm_debug_set", b"max_ctas", -1)


def test_epilogue_gelu_matches_fp64_erf():
    """The branch-free erf of the GEMM epilogue (sx_common.cuh erf_fast): |gelu - fp64 gelu| <= 4e-7 * max(1, |x|) over
    [-8, 8] — three orders below the TF32 operand rounding.  x is fed through an exact identity GEMM (TF32-exact inputs)."""
    from segtran_b200 import ops
    x = tf32(torch.linspace(-8, 8, 128 * 1024, device="cuda"))
    a = torch.zeros(x.numel(), 4, device="cuda")
    a[:, 0] = x
    y = ops.gemm_nt(a, torch.eye(4, device="cuda"), gelu=True, round_out=False)[0, 0, :, 0]
    ref = torch.nn.functional.gelu(x.double())
    err = (y.double() - ref).abs() / x.double().abs().clamp_min(1.0)
    assert float(err.max()) < 4e-7, float(err.max())


def test_gemm_gelu_bwd_epilogue_equals_separate_gelu_bwd_and_colsum():
    """SX_ACT_GELU_BWD: C = dropmask * (A B^T) * gelu'(h) in the GEMM epilogue == plain GEMM followed by sx_gelu_bwd with
    the same seed (bit-for-bit the same mask), and == the analytic fp64 expression when dropout is off."""
    import segtran_b200._lib as L
    from segtran_b200 import ops
    a = tf32(torch.randn(3, 200, 96, device="cuda"))
    b = tf32(torch.randn(3, 136, 96, device="cuda"))
    h = torch.randn(1, 3, 200, 136, device="cuda") * 2
    fused = ops.gemm_nt(a, b, gelu_bwd=h, round_out=False)
    hd = h.double()
    gp = 0.5 * (1 + torch.erf(hd / 2 ** 0.5)) + hd * torch.exp(-0.5 * hd * hd) / (2 * torch.pi) ** 0.5
    close(fused.double(), (a.double() @ b.double().transpose(-1, -2)).unsqueeze(0) * gp, 2e-6)
    seed = ops.new_dropout_seed(a.device)
    fused = ops.gemm_nt(a, b, gelu_bwd=h, drop_p=0.3, seed=seed, round_out=False)
    plain = ops.gemm_nt(a, b, round_out=False)
    sep = torch.empty_like(plain)
    L.call("sx_gelu_bwd", plain.data_ptr(), h.data_ptr(), plain.numel(), 0.3, 0, seed.data_ptr(), sep.data_ptr(), 0,
           torch.cuda.current_stream().cuda_stream)
    assert torch.equal(fused == 0, sep == 0)
    close(fused.double(), sep.double(), 1e-6)
    frac = float((fused == 0).float().mean())
    assert abs(frac - 0.3) < 0.01
    # column sums of the stored values (bias gradient), accumulated on top of what is already there
    cs = torch.ones(136, device="cuda")
    out = ops.gemm_nt(a, b, gelu_bwd=h, drop_p=0.3, seed=seed, round_out=False)
    ops.colsum(out.view(-1, 136), out=cs)
    close(cs.double(), 1.0 + out.double().sum(dim=(0, 1, 2)), 1e-5)


def test_linear_fwd_bwd_gelu():
    from segtran_b200 import ops
    x = torch.randn(5, 37, 96, device="cuda", requires_grad=True)
    W = torch.randn(128, 96, device="cuda", requires_grad=True) * 0.1
    W.retain_grad()
    b = torch.randn(128, device="cuda", requires_grad=True)
    y = ops.linear(x, W, b, gelu=True)
    g = torch.randn_like(y)
    y.backward(g)
    x2, W2, b2 = x.detach().clone().requires_grad_(), W.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
    y2 = F.gelu(F.linear(x2, W2, b2))
    y2.backward(g)
    close(y, y2, 2e-3)
    close(x.grad, x2.grad, 5e-3)
    close(W.grad, W2.grad, 5e-3)
    close(b.grad, b2.grad, 5e-3)


def test_softmax_matches_torch_and_dropout_statistics():
    from segtran_b200 import ops
    S = (torch.randn(3, 4, 50, 77, device="cuda") * 3).requires_grad_()
    P = ops.softmax(S)
    g = torch.randn_like(P)
    P.backward(g)
    S2 = S.detach().clone().requires_grad_()
    P2 = torch.softmax(S2, -1)
    P2.backward(g)
    close(P, P2, 1e-3)
    close(S.grad, S2.grad, 2e-3)
    # dropout: kept fraction ~ 1-p, kept values scaled by 1/(1-p), same mask regenerated in backward
    p = 0.3
    Sd = S.detach().clone().requires_grad_()
    Pd = ops.softmax(Sd, None, 500.0, p, 1234)
    kept = Pd != 0
    frac = float(kept.float().mean())
    assert abs(frac - (1 - p)) < 0.02, frac
    close(Pd[kept], (P2.detach() / (1 - p))[kept], 1e-3)
    Pd.backward(torch.ones_like(Pd))
    # d/dS of sum(dropout(P)): P * (m/(1-p) - sum_j P_j m_j/(1-p))
    m = kept.float() / (1 - p)
    ref = P2.detach() * (m - (P2.detach() * m).sum(-1, keepdim=True))
    close(Sd.grad, ref, 3e-3)


def test_clamp_only_when_global_max_exceeds_clip():
    from segtran_b200 import ops
    S = torch.randn(2, 1, 8, 40, device="cuda") * 100
    amax = S.max().reshape(1).clone()
    P = ops.softmax(S, amax, 50.0)
    close(P, torch.softmax(S.clamp(-50, 50), -1), 1e-3)
    P = ops.softmax(S, amax, 1e4)
    close(P, torch.softmax(S, -1), 1e-3)


def test_prologue_layernorm_and_aggregate():
    from segtran_b200 import ops
    B, N, C, C0, M = 2, 45, 96, 128, 4
    x = torch.randn(B, N, C, device="cuda", requires_grad=True)
    g = torch.randn(C, device="cuda", requires_grad=True)
    b = torch.randn(C, device="cuda", requires_grad=True)
    pe = torch.randn(N, C0, device="cuda", requires_grad=True)
    mask = (torch.rand(B * N, device="cuda") > 0.3).float()
    h = ops.prologue(x, g, b, pe, 1.0, mask)
    go = torch.randn_like(h)
    h.backward(go)
    xr, gr, br, per = [t.detach().clone().requires_grad_() for t in (x, g, b, pe)]
    t = F.layer_norm(xr, (C,), gr, br, 1e-12) + per[:, :C]
    hr = F.layer_norm(t, (C,), None, None, 1e-12) * mask.view(B, N, 1)
    hr.backward(go)
    close(h, hr, 1e-3)            # h is rounded to TF32 for the following GEMMs
    for a_, b_ in ((x.grad, xr.grad), (g.grad, gr.grad), (b.grad, br.grad), (pe.grad, per.grad)):
        close(a_, b_, 1e-4)
    # LN + soft aggregate
    Y = torch.randn(B, M, N, C, device="cuda", requires_grad=True)
    ws = torch.randn(1, C, device="cuda", requires_grad=True)
    bs = torch.randn(1, device="cuda", requires_grad=True)
    g2 = g.detach().clone().requires_grad_()
    b2 = b.detach().clone().requires_grad_()
    out = ops.ln_softaggr(Y, g2, b2, ws, bs)
    go = torch.randn_like(out)
    out.backward(go)
    Yr, g3, b3, wsr, bsr = [t.detach().clone().requires_grad_() for t in (Y, g2, b2, ws, bs)]
    yn = F.layer_norm(Yr, (C,), g3, b3, 1e-12)
    w = torch.softmax(F.linear(yn, wsr, bsr), dim=1)
    outr = (yn * w).sum(1)
    outr.backward(go)
    close(out, outr, 1e-5)
    close(Y.grad, Yr.grad, 1e-3)      # dY is rounded to TF32
    for a_, b_ in ((g2.grad, g3.grad), (b2.grad, b3.grad), (ws.grad, wsr.grad)):
        close(a_, b_, 1e-4)


def test_pos_code_fwd_bwd():
    from segtran_b200 import ops
    pos = torch.rand(70, 3, device="cuda") * 100
    W = torch.randn(64, 3, device="cuda", requires_grad=True)
    b = torch.randn(64, device="cuda", requires_grad=True)
    pe = ops.pos_code(pos, W, b)
    go = torch.randn_like(pe)
    pe.backward(go)
    Wr, br = W.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
    e = (pos / pos.max()) @ Wr.t() + br
    mix = torch.stack((torch.sin(e[:, 0::2]), torch.cos(e[:, 1::2])), dim=2).view(e.shape)
    per = F.layer_norm(mix, (64,), None, None, 1e-12)
    per.backward(go)
    close(pe, per, 1e-4)
    close(W.grad, Wr.grad, 1e-3)
    close(b.grad, br.grad, 1e-3)


@pytest.mark.parametrize("shape,size", [((2, 3, 5, 6, 7), (10, 12, 14)), ((2, 3, 5, 6, 7), (9, 6, 20)),
                                        ((2, 3, 4, 8, 12), (8, 16, 24)), ((1, 4, 8, 16), (16, 32)),    # x2 / float4 paths
                                        ((1, 2, 8, 9), (16, 27)), ((1, 2, 8, 9), (5, 9))])
def test_resize_linear_equals_interpolate(shape, size):
    from segtran_b200 import ops
    x = torch.randn(*shape, device="cuda", requires_grad=True)
    y = ops.resize_linear(x, size)
    go = torch.randn_like(y)
    y.backward(go)
    xr = x.detach().clone().requires_grad_()
    yr = F.interpolate(xr, size=size, mode="trilinear" if len(size) == 3 else "bilinear", align_corners=False)
    yr.backward(go)
    close(y, yr, 1e-5)
    close(x.grad, xr.grad, 1e-5)


def test_seg_head_3d_equals_uncollapsed():
    from segtran_b200 import ops
    B, Cf, Fd, K = 2, 24, 32, 4
    grid, sp1, out_size = (2, 3, 3), (4, 6, 6), (12, 12, 16)       # out_size = (H,W,D)
    curr = torch.randn(B, Cf, *sp1, device="cuda", requires_grad=True)
    vf = torch.randn(B, 18, Fd, device="cuda", requires_grad=True)
    Wb = torch.randn(Fd, Cf, 1, 1, 1, device="cuda", requires_grad=True)
    bb = torch.randn(Fd, device="cuda", requires_grad=True)
    Wc = torch.randn(K, Fd, 1, 1, 1, device="cuda", requires_grad=True)
    bc = torch.randn(K, device="cuda", requires_grad=True)
    y = ops.seg_head(curr, vf, grid, Wb, bb, Wc, bc, out_size, d_pool_k=2)
    go = torch.randn_like(y)
    y.backward(go)
    ts = [t.detach().clone().requires_grad_() for t in (curr, vf, Wb, bb, Wc, bc)]
    c2, v2, Wb2, bb2, Wc2, bc2 = ts
    up = F.interpolate(v2.transpose(1, 2).reshape(B, Fd, *grid), size=sp1, mode="trilinear", align_corners=False)
    x = F.conv3d(c2, Wb2, bb2) + up
    x = F.interpolate(x, size=(sp1[0] * 2, sp1[1], sp1[2]), mode="trilinear", align_corners=False)
    s = F.conv3d(x.permute(0, 1, 3, 4, 2), Wc2, bc2)
    yr = F.interpolate(s, size=out_size, mode="trilinear", align_corners=False)
    yr.backward(go)
    close(y, yr, 1e-4)                # forward is exact fp32 arithmetic (CUDA cores)
    for a_, b_ in zip((curr, vf, Wb, bb, Wc, bc), ts):
        close(a_.grad, b_.grad, 3e-3)  # weight gradients stream curr through the tensor cores as TF32


def test_seg_head_2d_odd_voxel_count_and_frozen_weights():
    """V = 7*9 is not a multiple of 4: the weight gradient takes the CUDA-core reduction (TMA needs 16-byte pitches);
    with every weight frozen no weight-gradient kernel runs and the data gradients are unchanged."""
    from segtran_b200 import ops
    B, Cf, Fd, K = 2, 16, 16, 3
    grid, sp1, out_size = (3, 4), (7, 9), (21, 27)
    for frozen in (False, True):
        torch.manual_seed(3)
        curr = torch.randn(B, Cf, *sp1, device="cuda", requires_grad=True)
        vf = torch.randn(B, 12, Fd, device="cuda", requires_grad=True)
        Wb = torch.randn(Fd, Cf, 1, 1, device="cuda", requires_grad=not frozen)
        bb = torch.randn(Fd, device="cuda", requires_grad=not frozen)
        Wc = torch.randn(K, Fd, 1, 1, device="cuda", requires_grad=not frozen)
        bc = torch.randn(K, device="cuda", requires_grad=not frozen)
        y = ops.seg_head(curr, vf, grid, Wb, bb, Wc, bc, out_size)
        go = torch.randn_like(y)
        y.backward(go)
        ts = [t.detach().clone().requires_grad_(t.requires_grad) for t in (curr, vf, Wb, bb, Wc, bc)]
        c2, v2, Wb2, bb2, Wc2, bc2 = ts
        up = F.interpolate(v2.transpose(1, 2).reshape(B, Fd, *grid), size=sp1, mode="bilinear", align_corners=False)
        s = F.conv2d(F.conv2d(c2, Wb2, bb2) + up, Wc2, bc2)
        yr = F.interpolate(s, size=out_size, mode="bilinear", align_corners=False)
        yr.backward(go)
        close(y, yr, 1e-4)
        for a_, b_ in zip((curr, vf, Wb, bb, Wc, bc), ts):
            if b_.requires_grad:
                close(a_.grad, b_.grad, 1e-4 if frozen else 3e-3)
            else:
                assert a_.grad is None
