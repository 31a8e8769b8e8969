"""Each dispatch branch of the row kernels (csrc/sx_rows.cu) against float64 PyTorch.  The dispatchers choose a kernel
by width, alignment and pitch: softmax fast NV = 2/4/8/16 (L % 4 == 0, L <= 2048), block E = 3/6/8 (L <= 3072 / 6144
/ 8192), warp + shared memory otherwise; the prologue's no-code warp kernel, CTA NV1/TT128, NV2/TT128, NV2/TT256 and
warp kernels; LayerNorm backward fast + column pass or warp; ln_softaggr CTA x M in {1, 2, 4} x three F tiers, or warp;
gelu_bwd float4 or scalar.  The widths sit on both sides of every threshold, one misaligned view (storage offset of one
float) forces the fallback at a width the fast path would take, and every case asserts by the kernel's name (recorded
by torch.profiler) that it ran the branch it names.  Tolerances are those of test_gpu_row_fallbacks.py; where the code
adds its column sums in a fixed order, two runs must agree bit for bit."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import assert_launched, close, close_on_scale, ln_softaggr64, prologue64, reference, run_twice

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def misaligned(t):
    """t's values in a contiguous view whose data pointer is one float past a 16-byte boundary (differentiable)"""
    return torch.cat([t.new_zeros(1), t.reshape(-1)])[1:].view(t.shape)


# ------------------------------------------------------------------------------------------------
# softmax with the conditional clamp: P, lse and dS (zero exactly where the clamp was active)
# ------------------------------------------------------------------------------------------------
def _softmax_kernel(Lr, aligned=True):
    if aligned and Lr % 4 == 0 and Lr <= 2048:
        nv = 2 if Lr <= 256 else 4 if Lr <= 512 else 8 if Lr <= 1024 else 16
        return "softmax_fwd_fast<%d>" % nv, "softmax_bwd_fast<%d>" % nv
    if aligned and Lr % 4 == 0 and Lr <= 8192:
        e = 3 if Lr <= 3072 else 6 if Lr <= 6144 else 8
        return "softmax_fwd_block<%d>" % e, "softmax_bwd_block<%d>" % e
    return "::softmax_fwd_kernel(", "::softmax_bwd_kernel("


def _softmax_run(S, R, Lr, ld, amax, clip):
    """forward and backward through the C ABI on R rows of pitch ld (all four operands), fixed upstream gradient"""
    from segtran_b200 import _lib as L
    P = torch.zeros_like(S)
    lse = torch.empty(R, device="cuda")
    G = torch.randn(R, Lr, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    dP = torch.zeros_like(S)
    dP.view(-1)[:R * ld].view(R, ld)[:, :Lr] = G
    dS = torch.zeros_like(S)
    L.call("sx_softmax_fwd", S.data_ptr(), R, Lr, ld, _ptr(amax), clip, 0.0, 0, None, P.data_ptr(), ld, 0, lse.data_ptr(),
           None, _stream())
    L.call("sx_softmax_bwd", dP.data_ptr(), ld, S.data_ptr(), ld, lse.data_ptr(), R, Lr, _ptr(amax), clip, 0.0, 0, None,
           ld, dS.data_ptr(), ld, 0, _stream())
    rows = lambda t: t.reshape(-1)[:R * ld].view(R, ld)[:, :Lr]      # noqa: E731
    return rows(P), lse, rows(dS), G


SOFTMAX_WIDTHS = [256, 260, 1024, 1028, 2048, 2052, 3072, 3076, 6144, 6148, 8192, 8196, 77]


@pytest.mark.parametrize("clamp", ["off", "below", "above"])
@pytest.mark.parametrize("Lr", SOFTMAX_WIDTHS)
def test_softmax_paths(Lr, clamp):
    """clamp: no amax; amax below the clip (no clamp); amax above it (scores beyond +-clip are clamped, their dS is 0)"""
    R = max(8, 262144 // Lr)
    ld = (Lr + 3) // 4 * 4
    S = torch.randn(R, ld, device="cuda") * 3
    clip = 4.0 if clamp == "above" else 500.0
    amax = None if clamp == "off" else S[:, :Lr].max().reshape(1)
    runs = [_softmax_run(S, R, Lr, ld, amax, clip) for _ in range(2)]
    P, lse, dS, G = runs[0]
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    S64 = S[:, :Lr].double()
    active = clamp == "above"
    Sc = S64.clamp(-clip, clip) if active else S64
    P64 = torch.softmax(Sc, -1)
    close(P, P64, 1e-5)
    close(lse, torch.logsumexp(Sc, -1), 1e-6)
    dS64 = P64 * (G.double() - (P64 * G.double()).sum(-1, keepdim=True))
    if active:
        outside = S64.abs() > clip
        assert bool(outside.any())
        assert bool((dS[outside] == 0).all())
        dS64 = dS64 * ~outside
    close(dS, dS64, 1e-4)
    assert_launched(lambda: _softmax_run(S, R, Lr, ld, amax, clip), *_softmax_kernel(Lr))


def test_softmax_misaligned_rows_take_the_warp_kernel():
    """L = 512 would take softmax_fwd_fast<4>; rows that start one float past a 16-byte boundary cannot"""
    Lr, R = 512, 300
    buf = torch.randn(R * Lr + 4, device="cuda") * 3
    S = buf[1:]
    run = lambda: _softmax_run(S, R, Lr, Lr, S[:R * Lr].max().reshape(1), 4.0)      # noqa: E731
    P, lse, dS, G = run()
    S64 = S[:R * Lr].view(R, Lr).double()
    P64 = torch.softmax(S64.clamp(-4.0, 4.0), -1)
    close(P, P64, 1e-5)
    close(lse, torch.logsumexp(S64.clamp(-4.0, 4.0), -1), 1e-6)
    inside = S64.abs() <= 4.0
    close(dS, P64 * (G.double() - (P64 * G.double()).sum(-1, keepdim=True)) * inside, 1e-4)
    assert bool((dS[~inside] == 0).all())
    assert_launched(run, *_softmax_kernel(Lr, aligned=False))


# ------------------------------------------------------------------------------------------------
# fused prologue: h, dx, dg, db, dpe
# ------------------------------------------------------------------------------------------------
def _prologue_kernel(C):
    nv, tt = (1, 128) if C <= 512 else (2, 128) if C <= 1024 else (2, 256)
    return "prologue_fwd_cta<%d,%d>" % (nv, tt), "prologue_bwd_cta<%d,%d>" % (nv, tt)


def _prologue_case(C, per_sample, kernels, mis=False):
    from segtran_b200 import ops
    B, N = 2, 300
    mask = (torch.rand(B * N, device="cuda") > 0.3).float()
    inputs = [torch.randn(B, N, C, device="cuda"), torch.randn(C, device="cuda"), torch.randn(C, device="cuda"),
              torch.randn(*((B,) if per_sample else ()), N, C, device="cuda")]
    h, grads = run_twice(
        lambda x, g, b, pe: ops.prologue(misaligned(x) if mis else x, g, b, pe, 0.7, mask), inputs, kernels=kernels)
    hr, grads_r = reference(lambda x, g, b, pe: prologue64(x, g, b, pe, 0.7, mask), inputs, h.shape)
    close(h, hr, 1e-3)            # h is rounded to TF32 for the following GEMMs
    for a, b in zip(grads, grads_r):
        close(a, b, 1e-4)


@pytest.mark.parametrize("C", [512, 516, 1024, 1028, 1540, 2044, 2048])
def test_prologue_cta_tiers(C):
    _prologue_case(C, per_sample=(C == 1540), kernels=_prologue_kernel(C))


def test_prologue_warp_kernels():
    """C = 2052 is wider than the CTA kernels' 2048; a misaligned x at C = 1024 cannot use them either"""
    warp = ("::prologue_fwd_kernel(", "::prologue_bwd_kernel(")
    _prologue_case(2052, per_sample=False, kernels=warp)
    _prologue_case(1024, per_sample=True, kernels=warp, mis=True)


@pytest.mark.parametrize("C", [98, 512, 2048])
def test_prologue_without_positional_code(C):
    from segtran_b200 import ops
    B, N = 2, 300
    mask = (torch.rand(B * N, device="cuda") > 0.3).float()
    inputs = [torch.randn(B, N, C, device="cuda"), torch.randn(C, device="cuda"), torch.randn(C, device="cuda")]
    h, grads = run_twice(lambda x, g, b: ops.prologue(x, g, b, None, 0.0, mask), inputs,
                         kernels=("prologue_nopos_fwd_kernel", "prologue_nopos_bwd_kernel"))
    hr, grads_r = reference(lambda x, g, b: prologue64(x, g, b, None, 0.0, mask), inputs, h.shape)
    close(h, hr, 1e-3)
    for a, b in zip(grads, grads_r):
        close(a, b, 1e-4)


# ------------------------------------------------------------------------------------------------
# LayerNorm backward: fast rows + column pass, or warp
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,mis,kernels", [
    (512, False, ("layernorm_bwd_rows_fast<4>", "ln_param_grad_cols_fast")),
    (516, False, ("layernorm_bwd_rows_fast<8>", "ln_param_grad_cols_fast")),
    (2048, False, ("layernorm_bwd_rows_fast<16>", "ln_param_grad_cols_fast")),
    (2052, False, ("::layernorm_bwd_kernel(",)),
    (512, True, ("::layernorm_bwd_kernel(",)),
])
def test_layernorm_backward_paths(C, mis, kernels):
    from segtran_b200 import ops
    R = 1500
    inputs = [torch.randn(R, C, device="cuda"), torch.randn(C, device="cuda"), torch.randn(C, device="cuda")]
    y, grads = run_twice(lambda x, g, b: ops.layer_norm(misaligned(x) if mis else x, g, b), inputs, kernels=kernels)
    yr, grads_r = reference(lambda x, g, b: F.layer_norm(x, (C,), g, b, 1e-12), inputs, y.shape)
    close(y, yr, 1e-3)            # y and dx are rounded to TF32 for the neighbouring GEMMs
    close(grads[0], grads_r[0], 1e-3)
    for a, b in zip(grads[1:], grads_r[1:]):
        close(a, b, 1e-4)


# ------------------------------------------------------------------------------------------------
# LayerNorm + soft aggregation: out, dY, dg, db, dws, dbs
# ------------------------------------------------------------------------------------------------
def _lnsa_case(M, F_, kernels, mis=False):
    from segtran_b200 import ops
    B, N = 2, 128
    inputs = [torch.randn(B, M, N, F_, device="cuda"), torch.randn(F_, device="cuda"), torch.randn(F_, device="cuda"),
              torch.randn(1, F_, device="cuda") * 0.05, torch.randn(1, device="cuda")]
    out, grads = run_twice(
        lambda Y, g, b, ws, bs: ops.ln_softaggr(misaligned(Y) if mis else Y, g, b, ws, bs), inputs, kernels=kernels)
    outr, grads_r = reference(ln_softaggr64, inputs, out.shape)
    close(out, outr, 1e-5)
    close(grads[0], grads_r[0], 1e-3)      # dY is rounded to TF32
    for a, b in zip(grads[1:4], grads_r[1:4]):
        close(a, b, 1e-4)
    # d bs is a sum of score gradients whose sum over the modes of each token is zero: compare on the scale of d ws
    close_on_scale(grads[4], grads_r[4], float(grads_r[3].abs().max()), 1e-4)      # (M = 1: both exactly 0)


LNSA_CTA = [(4, F_) for F_ in (512, 516, 1024, 1028, 1540, 2044, 2048)] + \
           [(M, F_) for M in (1, 2) for F_ in (512, 1024, 1540)]


@pytest.mark.parametrize("M,F_", LNSA_CTA)
def test_ln_softaggr_cta_paths(M, F_):
    nv, tt = (1, 128) if F_ <= 512 else (2, 128) if F_ <= 1024 else (2, 256)
    _lnsa_case(M, F_, ("ln_softaggr_fwd_cta<%d,%d,%d>" % (nv, M, tt), "ln_softaggr_bwd_cta<%d,%d,%d>" % (nv, M, tt)))


@pytest.mark.parametrize("M,F_,mis", [(3, 512, False), (4, 1024, True)])
def test_ln_softaggr_warp_paths(M, F_, mis):
    """M = 3 modes has no CTA form; a misaligned Y at M = 4, F = 1024 cannot use it either"""
    _lnsa_case(M, F_, ("::ln_softaggr_fwd_kernel(", "::ln_softaggr_bwd_kernel("), mis)


# ------------------------------------------------------------------------------------------------
# gelu_bwd without dropout: float4 and scalar kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,off,kernel", [(4096 * 9, 0, "gelu_bwd_f4_kernel<true>"), (4096 * 9 + 1, 0, "gelu_bwd_kernel<true>"),
                                          (4096 * 9, 1, "gelu_bwd_kernel<true>")])
def test_gelu_bwd_paths(n, off, kernel):
    from segtran_b200 import _lib as L
    dG = torch.randn(n + off, device="cuda")[off:]
    H = (torch.randn(n + off, device="cuda") * 3)[off:]
    dH = torch.empty(n + off, device="cuda")[off:]
    run = lambda: L.call("sx_gelu_bwd", dG.data_ptr(), H.data_ptr(), n, 0.0, 0, None, dH.data_ptr(), 0, _stream())  # noqa: E731
    run()
    h = H.double()
    gp = 0.5 * (1 + torch.erf(h / math.sqrt(2))) + h * torch.exp(-0.5 * h * h) / math.sqrt(2 * math.pi)
    close(dH, dG.double() * gp, 1e-5)
    assert_launched(run, kernel)
