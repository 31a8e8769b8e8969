"""Every dropout site against the exact host mask.  No mask is ever stored: each site hashes (seed, flat element index)
with the counter-based hash of csrc/sx_common.cuh, and the backward hashes again.  Here each site's mask is made visible
(an output or a gradient that is exactly zero where an element was dropped) and must equal, element for element, the mask
that oracle/head_oracle.py:drop_keep1 computes on the host at the index convention the site documents:

  softmax / posbias softmax / fused attention   r * ldp + c   (r the flattened row, ldp P's padded row pitch)
  GEMM epilogue                                 zoff + row * ldc + col
  prologue                                      r * C + c
  ln_softaggr                                   the flat index of Y [B, M, N, F]
  gelu_bwd                                      the flat index i from the dG pointer

The backward of each site is then compared with a float64 reference built from the host mask, so a backward that
regenerates a different mask (another index, another seed, another 16-bit field) is off by O(1).  The statistical
checks of test_gpu_dropout_sites.py pass for such a mask; these do not."""
import math

import pytest
import torch

from tests.helpers import assert_launched, close, close_on_scale, host_keep, ln_softaggr64, pitched_index, prologue64

pytestmark = pytest.mark.gpu

P_NEAR_1 = 1 - 2 ** -17       # p * 65536 + 0.5 = 65536: drop_p16 clamps it to 65535 (one element in 65536 is kept);
                              # 1 - p is exact in fp32, so the kernels' keep scale is exactly 1 / (1 - p)
NEAR_1_ELEMENTS = 1 << 21     # the p = P_NEAR_1 cases span this many elements or more: some 32 of them are kept


def near_1_rows(p, rows, cols):
    """rows, or enough rows of `cols` elements for NEAR_1_ELEMENTS when p = P_NEAR_1"""
    return max(rows, -(-NEAR_1_ELEMENTS // cols)) if p == P_NEAR_1 else rows


@pytest.fixture(autouse=True)
def _fp32_grade_precision():
    """tf32x3 mode: no kernel rounds its output to TF32, so kept values compare with the fp64 reference at fp32 accuracy"""
    from segtran_b200 import ops
    torch.manual_seed(0)
    ops.set_precision("tf32x3")
    yield
    ops.set_precision("tf32")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _pad4(n):
    return (n + 3) // 4 * 4


def gelu_grad64(h):
    h = h.double()
    return 0.5 * (1 + torch.erf(h / math.sqrt(2))) + h * torch.exp(-0.5 * h * h) / math.sqrt(2 * math.pi)


def softmax_bwd64(P0, g):
    """dS of softmax with upstream gradient g (float64)"""
    return P0 * (g - (P0 * g).sum(-1, keepdim=True))


def check_mask(visible, keep, p=None):
    """visible: the values that are exactly zero where dropped (nonzero elsewhere).  The host mask must keep elements
    (at p = P_NEAR_1 at least 8), or the comparison could not see the index."""
    assert int(keep.sum()) >= (8 if p == P_NEAR_1 else 1), int(keep.sum())
    dropped = visible == 0
    assert torch.equal(dropped, ~keep), "mask differs from the host mask at %d of %d elements" % (
        int((dropped != ~keep).sum()), keep.numel())


# ------------------------------------------------------------------------------------------------
# softmax (sx_softmax_fwd / sx_softmax_bwd), called directly so that every pitch is explicit
# ------------------------------------------------------------------------------------------------
def _pitched(rows, cols, ld, scale=2.0):
    return (torch.randn(rows, ld, device="cuda") * scale)[:, :cols]


def softmax_fwd(S, ldp, p, seed, seed_dev=None):
    from segtran_b200 import _lib as L
    R, Lr = S.shape
    Pb = torch.zeros(R, ldp, device="cuda")
    lse = torch.empty(R, device="cuda")
    L.call("sx_softmax_fwd", S.data_ptr(), R, Lr, S.stride(0), None, 500.0, p, seed, _ptr(seed_dev), Pb.data_ptr(), ldp,
           0, lse.data_ptr(), None, _stream())
    return Pb[:, :Lr], lse


def softmax_bwd(dP, S, lse, ldp_fwd, ldo, p, seed, seed_dev=None):
    from segtran_b200 import _lib as L
    R, Lr = S.shape
    dSb = torch.zeros(R, ldo, device="cuda")
    L.call("sx_softmax_bwd", dP.data_ptr(), dP.stride(0), S.data_ptr(), S.stride(0), lse.data_ptr(), R, Lr, None, 500.0,
           p, seed, _ptr(seed_dev), ldp_fwd, dSb.data_ptr(), ldo, 0, _stream())
    return dSb[:, :Lr]


# (L, P's pitch ldp, dS's pitch ldo, forward kernel, backward kernel).  ldp > L pads P; ldo % 4 != 0 sends the backward
# of a fast-path forward to the warp kernel, so the two regenerate the mask on different paths.
SOFTMAX_CASES = [
    (512, 512, 512, "softmax_fwd_fast<4>", "softmax_bwd_fast<4>"),
    (256, 260, 256, "softmax_fwd_fast<2>", "softmax_bwd_fast<2>"),
    (512, 512, 513, "softmax_fwd_fast<4>", "::softmax_bwd_kernel("),
    (3072, 3072, 3072, "softmax_fwd_block<3>", "softmax_bwd_block<3>"),
    (3076, 3080, 3076, "softmax_fwd_block<6>", "softmax_bwd_block<6>"),
    (8196, 8196, 8196, "::softmax_fwd_kernel(", "::softmax_bwd_kernel("),
    (77, 80, 80, "::softmax_fwd_kernel(", "::softmax_bwd_kernel("),
]


@pytest.mark.parametrize("p", [0.3, 0.5, P_NEAR_1])
@pytest.mark.parametrize("Lr,ldp,ldo,kfwd,kbwd", SOFTMAX_CASES)
def test_softmax_mask_is_the_host_mask(Lr, ldp, ldo, kfwd, kbwd, p):
    R = near_1_rows(p, max(16, 131072 // Lr), Lr)
    seed = 0x9E3779B97F4A7C15 + Lr
    S = _pitched(R, Lr, _pad4(Lr))
    G = _pitched(R, Lr, _pad4(Lr), 1.0)
    P, lse = softmax_fwd(S, ldp, p, seed)
    keep = host_keep(seed, pitched_index(R, Lr, ldp), p)
    check_mask(P, keep, p)
    P0 = torch.softmax(S.double(), -1)
    close(P[keep], P0[keep] / (1 - p), 1e-5)
    close(lse, torch.logsumexp(S.double(), -1), 1e-6)
    dS = softmax_bwd(G, S, lse, ldp, ldo, p, seed)
    close(dS, softmax_bwd64(P0, G.double() * keep / (1 - p)), 1e-4)
    assert_launched(lambda: softmax_fwd(S, ldp, p, seed), kfwd)
    assert_launched(lambda: softmax_bwd(G, S, lse, ldp, ldo, p, seed), kbwd)


@pytest.mark.parametrize("Lr,ldp", [(512, 512), (3072, 3076), (77, 80)])
def test_softmax_adds_the_device_seed_to_the_seed_value(Lr, ldp):
    """seed_dev is the per-call device seed of a captured graph: the kernels hash with seed + *seed_dev"""
    R = 64
    a, b = 0x0123456789ABCDEF, 0xFEDCBA9876543210
    seed_dev = torch.tensor([b - (1 << 64)], dtype=torch.int64, device="cuda")
    S = _pitched(R, Lr, _pad4(Lr))
    G = _pitched(R, Lr, _pad4(Lr), 1.0)
    P, lse = softmax_fwd(S, ldp, 0.5, a, seed_dev)
    keep = host_keep(a + b, pitched_index(R, Lr, ldp), 0.5)
    check_mask(P, keep)
    dS = softmax_bwd(G, S, lse, ldp, _pad4(Lr), 0.5, a, seed_dev)
    close(dS, softmax_bwd64(torch.softmax(S.double(), -1), G.double() * keep / 0.5), 1e-4)


def test_softmax_autograd_node():
    """ops.softmax over a 4-D score tensor of odd width (P row-padded to 80): the node's own pitch and seed plumbing"""
    from segtran_b200 import ops
    seed, p = 424242, 0.3
    S = (torch.randn(2, 3, 50, 77, device="cuda") * 2).requires_grad_()
    P = ops.softmax(S, None, 500.0, p, seed)
    keep = host_keep(seed, pitched_index(2 * 3 * 50, 77, P.stride(-2)), p).view(P.shape)
    check_mask(P.detach(), keep)
    G = torch.randn_like(P)
    P.backward(G)
    P0 = torch.softmax(S.detach().double(), -1)
    close(S.grad, softmax_bwd64(P0, G.double() * keep / (1 - p)), 1e-4)


# ------------------------------------------------------------------------------------------------
# softmax with the sliding-window positional bias
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid,R", [((7, 9), 2), ((3, 4, 5), 1)])
def test_posbias_softmax_mask_is_the_host_mask(grid, R):
    from oracle.posbias_oracle import dense_bias
    from segtran_b200 import ops
    seed, p, w, M = 77, 0.5, 0.8, 2
    N = math.prod(grid)
    table = (torch.randn([2 * R + 1] * len(grid), device="cuda") * 0.7).requires_grad_()
    S = (torch.randn(1, M, N, N, device="cuda") * 2).requires_grad_()
    run = lambda: ops.softmax(S, None, 500.0, p, seed, posbias=ops.PosBias(table, R, grid, w))     # noqa: E731
    P = run()
    keep = host_keep(seed, pitched_index(M * N, N, P.stride(-2)), p).view(P.shape)
    check_mask(P.detach(), keep)
    G = torch.randn_like(P)
    P.backward(G)
    S64 = S.detach().double().requires_grad_()
    T64 = table.detach().double().cpu().requires_grad_()
    P64 = torch.softmax(S64 + w * dense_bias(T64, R, grid).cuda(), -1)
    close(P.detach()[keep], P64.detach()[keep] / (1 - p), 1e-5)
    (P64 * G.double() * keep / (1 - p)).sum().backward()
    close(S.grad, S64.grad, 1e-4)
    close(table.grad, T64.grad, 1e-4)
    assert_launched(lambda: torch.autograd.grad(run(), (S, table), G), "softmax_posbias_fwd_kernel",
                    "softmax_posbias_bwd_kernel")


# ------------------------------------------------------------------------------------------------
# fused attention probabilities (sx_attn.cu): ((b*M + m)*U1 + row)*ldp + col
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,U2", [(1, 77), (4, 77), (1, 300), (4, 300)])
def test_fused_attention_mask_is_the_host_mask(M, U2):
    """U2 = 77: P's rows padded to 80; U2 = 300 > 128: the kernel's two passes over the key tiles"""
    from segtran_b200 import ops
    B, U1, d, p, seed = 2, 70, 16, 0.3, 0xC0FFEE + U2
    q = torch.randn(B, U1, M * d, device="cuda")
    k = torch.randn(B, U2, M * d, device="cuda")
    run = lambda: ops.attn_probs_fused(q, k, M, 500.0, p, seed, need_scores=True, round_out=False)   # noqa: E731
    P, S, lse, _rowmax, stat = run()
    ldp = P.stride(-2)
    keep = host_keep(seed, pitched_index(B * M * U1, U2, ldp), p).view(P.shape)
    check_mask(P, keep)
    P0 = torch.softmax(S.double(), -1)
    close(P[keep], P0[keep] / (1 - p), 1e-5)
    G = torch.randn(B, M, U1, U2, device="cuda")
    dS, _ = ops.softmax_backward(G, S, lse, stat[2:], 500.0, p, seed, ldp)
    close(dS, softmax_bwd64(P0, G.double() * keep / (1 - p)), 1e-4)
    assert_launched(run, "sx_attn_probs_kernel<false,false>")


# ------------------------------------------------------------------------------------------------
# GEMM epilogue (sx_gemm.cu): zoff + row*ldc + col, per-thread words when (ldc | zoff) % 4 == 0, scalar hashes otherwise
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.3, P_NEAR_1])
@pytest.mark.parametrize("act", ["none", "gelu_bwd"])
@pytest.mark.parametrize("wide", [0, 1])
@pytest.mark.parametrize("ldc_pad", [0, 1])
def test_gemm_epilogue_mask_is_the_host_mask(ldc_pad, wide, act, p):
    """ldc_pad = 1: odd ldc (a strided out), the scalar hash path; wide = 1: the 128 x 256 tile"""
    from segtran_b200 import _lib as L, ops
    Z0, N, K, seed = 2, 264, 64, 31337 + 2 * ldc_pad + wide
    ldc = N + ldc_pad
    M = near_1_rows(p, 200, Z0 * N)
    a = torch.randn(1, Z0, M, K, device="cuda")
    b = torch.randn(Z0, N, K, device="cuda") * 0.2
    out = torch.zeros(Z0, M, ldc, device="cuda")[..., :N]
    h = (torch.randn(Z0, M, ldc, device="cuda") * 2)[..., :N] if act == "gelu_bwd" else None

    def run():
        try:
            L.call("sx_gemm_debug_set", b"wide_tiles", wide)
            ops.gemm_nt(a, b, out=out, drop_p=p, seed=seed, round_out=False, gelu_bwd=h)
            torch.cuda.synchronize()
        finally:
            L.call("sx_gemm_debug_set", b"wide_tiles", -1)
    run()
    idx = torch.arange(Z0 * M * ldc, device="cuda").view(Z0, M, ldc)[..., :N]
    keep = host_keep(seed, idx, p)
    check_mask(out, keep, p)
    ref = (a[0].double() @ b.double().transpose(-1, -2)) * keep / (1 - p)
    if h is not None:
        ref = ref * gelu_grad64(h)
    close(out, ref, 1e-5)
    assert_launched(run, "sx_gemm_kernel<4,false,false,%d>" % (256 if wide else 128))


# ------------------------------------------------------------------------------------------------
# fused prologue: r*C + c, with and without the positional code
# ------------------------------------------------------------------------------------------------
PROLOGUE_CASES = [                            # (C, positional code, forward kernel, backward kernel)
    (96, False, "prologue_nopos_fwd_kernel", "prologue_nopos_bwd_kernel"),
    (512, True, "prologue_fwd_cta<1,128>", "prologue_bwd_cta<1,128>"),
    (1024, True, "prologue_fwd_cta<2,128>", "prologue_bwd_cta<2,128>"),
    (2048, True, "prologue_fwd_cta<2,256>", "prologue_bwd_cta<2,256>"),
    (98, True, "::prologue_fwd_kernel(", "::prologue_bwd_kernel("),
]


@pytest.mark.parametrize("p", [0.3, P_NEAR_1])
@pytest.mark.parametrize("C,with_pe,kfwd,kbwd", PROLOGUE_CASES)
def test_prologue_mask_is_the_host_mask(C, with_pe, kfwd, kbwd, p):
    from segtran_b200 import ops
    B, posw, seed = 2, 0.7, 987654321 + C
    N = near_1_rows(p, 300, B * C)
    x = torch.randn(B, N, C, device="cuda", requires_grad=True)
    g = (1 + 0.1 * torch.randn(C, device="cuda")).requires_grad_()
    b = (0.1 * torch.randn(C, device="cuda")).requires_grad_()
    pe = torch.randn(N, C, device="cuda", requires_grad=True) if with_pe else None
    mask = torch.ones(B * N, device="cuda")
    run = lambda: ops.prologue(x, g, b, pe, posw if with_pe else 0.0, mask, p, seed)       # noqa: E731
    h = run()
    keep = host_keep(seed, pitched_index(B * N, C, C), p).view(B, N, C)
    check_mask(h.detach(), keep, p)
    G = torch.randn_like(h)
    h.backward(G)
    leaves = [t for t in (x, g, b, pe) if t is not None]
    l64 = [t.detach().double().requires_grad_() for t in leaves]
    h64 = prologue64(*l64[:3], l64[3] if with_pe else None, posw, keep=keep, p=p)
    close(h.detach(), h64.detach(), 1e-5)
    (h64 * G.double()).sum().backward()
    for a_, r_ in zip(leaves, l64):
        close(a_.grad, r_.grad, 1e-4)
    assert_launched(lambda: torch.autograd.grad(run(), leaves, G), kfwd, kbwd)


# ------------------------------------------------------------------------------------------------
# LayerNorm + soft aggregation over modes: the flat index of Y
# ------------------------------------------------------------------------------------------------
LNSA_CASES = [                                # (M, F, forward kernel, backward kernel)
    (1, 512, "ln_softaggr_fwd_cta<1,1,128>", "ln_softaggr_bwd_cta<1,1,128>"),
    (2, 1024, "ln_softaggr_fwd_cta<2,2,128>", "ln_softaggr_bwd_cta<2,2,128>"),
    (4, 2048, "ln_softaggr_fwd_cta<2,4,256>", "ln_softaggr_bwd_cta<2,4,256>"),
    (3, 96, "::ln_softaggr_fwd_kernel(", "::ln_softaggr_bwd_kernel("),
]


@pytest.mark.parametrize("p", [0.3, 0.5])
@pytest.mark.parametrize("M,F_,kfwd,kbwd", LNSA_CASES)
def test_ln_softaggr_mask_is_the_host_mask(M, F_, kfwd, kbwd, p):
    from segtran_b200 import ops
    B, N, seed = 2, 150, 5550123 + M
    leaves = [torch.randn(B, M, N, F_, device="cuda"), 1 + 0.1 * torch.randn(F_, device="cuda"),
              0.1 * torch.randn(F_, device="cuda"), torch.randn(1, F_, device="cuda") * 0.05,
              torch.randn(1, device="cuda")]
    leaves = [t.requires_grad_() for t in leaves]
    run = lambda: ops.ln_softaggr(*leaves, p, seed)                 # noqa: E731
    out = run()
    G = torch.randn_like(out)
    out.backward(G)
    keep = host_keep(seed, torch.arange(B * M * N * F_, device="cuda"), p).view(B, M, N, F_)
    check_mask(leaves[0].grad, keep)
    Y, g, b, ws, bs = [t.detach().double().requires_grad_() for t in leaves]
    out64 = ln_softaggr64(Y, g, b, ws, bs, keep, p)
    close(out.detach(), out64.detach(), 1e-5)
    (out64 * G.double()).sum().backward()
    for a_, r_ in zip(leaves[:4], (Y, g, b, ws)):
        close(a_.grad, r_.grad, 1e-4)
    # d bs sums score gradients whose sum over the modes is zero per token: compare on the scale of d ws
    close_on_scale(leaves[4].grad, bs.grad, float(ws.grad.abs().max()), 1e-4)        # (M = 1: both exactly 0)
    assert_launched(lambda: torch.autograd.grad(run(), leaves, G), kfwd, kbwd)


# ------------------------------------------------------------------------------------------------
# gelu_bwd (the backward of a GEMM epilogue's dropout, with or without GELU): the flat index from the dG pointer
# ------------------------------------------------------------------------------------------------
GELU_CASES = [                                # (n, element offset of every pointer, GELU, kernel)
    (4096 * 33, 0, True, "gelu_bwd_f4_kernel<true>"),
    (4096 * 33, 0, False, "gelu_bwd_f4_kernel<false>"),
    (4097 * 33, 0, True, "gelu_bwd_kernel<true>"),
    (4096 * 33, 1, True, "gelu_bwd_kernel<true>"),
    (4097 * 33, 0, False, "gelu_bwd_kernel<false>"),
]


@pytest.mark.parametrize("p", [0.3, 0.5, P_NEAR_1])
@pytest.mark.parametrize("n,off,gelu,kernel", GELU_CASES)
def test_gelu_bwd_mask_is_the_host_mask(n, off, gelu, kernel, p):
    from segtran_b200 import _lib as L
    seed = 0xA5A5A5A5A5A5 + n + off
    if p == P_NEAR_1:                         # 16 times the elements; n % 4, so the kernel, unchanged
        n += 15 * 4096 * 33
    dG = torch.randn(n + off, device="cuda")[off:]
    H = (torch.randn(n + off, device="cuda") * 2)[off:] if gelu else None
    dH = torch.zeros(n + off, device="cuda")[off:]
    run = lambda: L.call("sx_gelu_bwd", dG.data_ptr(), _ptr(H), n, p, seed, None, dH.data_ptr(), 0, _stream())  # noqa: E731
    run()
    keep = host_keep(seed, torch.arange(n, device="cuda"), p)
    check_mask(dH, keep, p)
    ref = dG.double() * keep / (1 - p)
    close(dH, ref * gelu_grad64(H) if gelu else ref, 1e-5)
    assert_launched(run, kernel)


def test_gelu_bwd_adds_the_device_seed_to_the_seed_value():
    from segtran_b200 import _lib as L
    n, a, b = 4096 * 8 + 3, 12345, (1 << 63) + 977
    seed_dev = torch.tensor([b - (1 << 64)], dtype=torch.int64, device="cuda")
    for off in (0, 3):                        # scalar kernel (n odd), then f4 kernel on n - 3 aligned elements
        m = n - off
        dG = torch.randn(m, device="cuda")
        dH = torch.empty(m, device="cuda")
        L.call("sx_gelu_bwd", dG.data_ptr(), None, m, 0.5, a, seed_dev.data_ptr(), dH.data_ptr(), 0, _stream())
        check_mask(dH, host_keep(a + b, torch.arange(m, device="cuda"), 0.5))
