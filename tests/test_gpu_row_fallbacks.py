"""The generic row and reduction kernels: the paths for odd widths, widths above 2048, mode counts other than 1, 2, 4
and odd voxel counts.  Each is checked against fp64 PyTorch at the tolerances of test_gpu_ops.py, and two calls on the
same inputs must give bit-identical outputs and gradients (every cross-CTA sum is added in a fixed order)."""

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import close, close_on_scale, ln_softaggr64, prologue64, reference, run_twice

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.mark.parametrize("C,C0,per_sample", [(98, 128, False), (2056, 2056, True)])
def test_prologue_with_positional_code(C, C0, per_sample):
    """C = 98 is not a multiple of 4 and C = 2056 is wider than the CTA kernel's 2048: both take the warp-per-row kernel,
    whose dpe comes from dt through the ordered column pass."""
    from segtran_b200 import ops
    B, N = 2, 700
    mask = (torch.rand(B * N, device="cuda") > 0.3).float()
    inputs = [torch.randn(B, N, C, device="cuda"), torch.randn(C, device="cuda"), torch.randn(C, device="cuda"),
              torch.randn(*((B,) if per_sample else ()), N, C0, device="cuda")]
    h, grads = run_twice(lambda x, g, b, pe: ops.prologue(x, g, b, pe, 0.7, mask), inputs)

    hr, grads_r = reference(lambda x, g, b, pe: prologue64(x, g, b, pe, 0.7, mask), inputs, h.shape)
    close(h, hr, 1e-3)            # h is rounded to TF32 for the following GEMMs
    for a, b in zip(grads, grads_r):
        close(a, b, 1e-4)


def test_layernorm_odd_width():
    from segtran_b200 import ops
    R, C = 1500, 97
    inputs = [torch.randn(R, C, device="cuda"), torch.randn(C, device="cuda"), torch.randn(C, device="cuda")]
    y, grads = run_twice(ops.layer_norm, inputs)
    yr, grads_r = reference(lambda x, g, b: F.layer_norm(x, (C,), g, b, 1e-12), inputs, y.shape)
    close(y, yr, 1e-3)            # y and dx are rounded to TF32 for the neighbouring GEMMs
    close(grads[0], grads_r[0], 1e-3)
    for a, b in zip(grads[1:], grads_r[1:]):
        close(a, b, 1e-4)


@pytest.mark.parametrize("M,F_", [(3, 96), (4, 98)])
def test_ln_softaggr_generic(M, F_):
    """M = 3 modes, and F = 98 (not a multiple of 4) with 4 modes: the warp-per-token kernel."""
    from segtran_b200 import ops
    B, N = 2, 600
    inputs = [torch.randn(B, M, N, F_, device="cuda"), torch.randn(F_, device="cuda"), torch.randn(F_, device="cuda"),
              torch.randn(1, F_, device="cuda"), torch.randn(1, device="cuda")]
    out, grads = run_twice(ops.ln_softaggr, inputs)

    outr, grads_r = reference(ln_softaggr64, inputs, out.shape)
    close(out, outr, 1e-5)
    close(grads[0], grads_r[0], 1e-3)      # dY is rounded to TF32
    for a, b in zip(grads[1:4], grads_r[1:4]):
        close(a, b, 1e-4)
    # d bs is a sum of score gradients whose sum over the modes of each token is zero: compare on the scale of d ws
    close_on_scale(grads[4], grads_r[4], float(grads_r[3].abs().max()), 1e-4)


def test_colsum_odd_width():
    from segtran_b200 import _lib as L, ops
    x = torch.randn(3000, 37, device="cuda")
    sums = [ops.colsum(x) for _ in range(2)]
    assert torch.equal(sums[0], sums[1])
    close(sums[0], x.double().sum(0), 1e-5)
    # batched: X [Z1=2][Z0=3][R][C] -> out [Z0][C], accumulated on top of what is there
    X = torch.randn(2, 3, 900, 37, device="cuda")
    outs = []
    for _ in range(2):
        out = torch.ones(3 * 37, device="cuda")
        L.call("sx_colsum_batched", X.data_ptr(), 2, X.stride(0), 3, X.stride(1), 900, 37, 37, out.data_ptr(),
               *ops._part_args(X.device), torch.cuda.current_stream().cuda_stream)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    close(outs[0], 1.0 + X.double().sum(dim=(0, 2)).reshape(-1), 1e-5)


def test_dot_is_ordered():
    from segtran_b200 import ops
    x, w = torch.randn(3, 1001, 77, device="cuda"), torch.randn(3, 1001, 77, device="cuda")
    vals = [ops.dot(x, w) for _ in range(2)]
    assert torch.equal(vals[0], vals[1])
    close(vals[0], (x.double() * w.double()).sum().view(1), 1e-5)


def test_head_weight_gradient_odd_voxel_count():
    """V = 7*9*5 is not a multiple of 4: the class weights' gradient is the CUDA-core reduction with per-CTA slots."""
    from segtran_b200 import ops
    B, Cf, Fd, K = 2, 16, 16, 3
    grid, sp1, out_size = (3, 4, 2), (7, 9, 5), (14, 18, 15)
    inputs = [torch.randn(B, Cf, *sp1, device="cuda"), torch.randn(B, 24, Fd, device="cuda"),
              torch.randn(Fd, Cf, 1, 1, 1, device="cuda"), torch.randn(Fd, device="cuda"),
              torch.randn(K, Fd, 1, 1, 1, device="cuda"), torch.randn(K, device="cuda")]
    y, grads = run_twice(lambda *t: ops.seg_head(*t[:2], grid, *t[2:], out_size), inputs)

    def ref(curr, vf, Wb, bb, Wc, bc):
        up = F.interpolate(vf.transpose(1, 2).reshape(B, Fd, *grid), size=sp1, mode="trilinear", align_corners=False)
        s = F.conv3d(F.conv3d(curr, Wb, bb) + up, Wc, bc).permute(0, 1, 3, 4, 2)
        return F.interpolate(s, size=out_size, mode="trilinear", align_corners=False)
    yr, grads_r = reference(ref, inputs, y.shape)
    close(y, yr, 1e-4)
    for a, b in zip(grads, grads_r):
        close(a, b, 3e-3)
