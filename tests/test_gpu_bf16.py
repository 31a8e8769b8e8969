"""The bf16-operand tensor-core mode (ops.set_precision("bf16"), BASELINE.json config 5's precision): every operand
majorness of the GEMM against an fp64 product of the bf16-rounded operands, and the
encoder fixtures forward + backward within the mode's error budget."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K,Z", [(520, 512, 256, 3), (96, 264, 1024, 2), (2744, 1024, 1024, 2)])
def test_gemm_bf16_operands_all_majors(M, N, K, Z):
    from segtran_b200 import ops
    torch.manual_seed(M)
    a = torch.randn(Z, 1, M, K, device="cuda")
    b = torch.randn(Z, 1, N, K, device="cuda")
    ar, br = a.bfloat16().double(), b.bfloat16().double()
    ref = ar @ br.transpose(-1, -2)
    am = a.transpose(-1, -2).contiguous().transpose(-1, -2)
    bm = b.transpose(-1, -2).contiguous().transpose(-1, -2)
    ops.set_precision("bf16")
    try:
        for x, y in ((a, b), (am, bm), (a, bm), (am, b)):
            c = ops.gemm_nt(x, y)
            assert rel_err(c, ref) < 2e-5            # exact products of bf16 values, fp32 accumulation
        red = ops.gemm_nt(a, b, reduce_z1=True)
        assert rel_err(red[0], ref.sum(0)) < 2e-5
    finally:
        ops.set_precision("tf32")


def test_small_encoder_in_bf16_mode_vs_oracle():
    """forward + input gradient of a small stack (token count and widths multiples of 8: bf16 TMA row pitches are 16 bytes)
    against the fp32 oracle, within the mode's budget."""
    from oracle import segtran_oracle as O
    from segtran_b200 import ops
    from tests.test_gpu_fullsize_configs import _build
    dims, A, grid = [64, 64], 16, (4, 4, 4)
    enc = _build(dims, A, grid, True, seed=3).eval()
    p = {"voxel_fusion." + k: v.clone() for k, v in enc.state_dict().items() if ".key." not in k}
    torch.manual_seed(4)
    x = torch.randn(2, 64, 64)
    pos = O.voxels_pos_for_grid(grid, (8, 8, 8), 2)
    mask = torch.ones(2, 64, 1)
    G = torch.randn(2, 64, 64)
    xr = x.clone().requires_grad_()
    ref = O.fusion_encoder(p, "voxel_fusion.", xr, pos, mask, dims, 4)
    (ref * G).sum().backward()
    enc = enc.cuda()
    xg = x.cuda().requires_grad_()
    ops.set_precision("bf16")
    try:
        y = enc(xg, pos.cuda(), mask.cuda(), torch.Size(grid))
        (y * G.cuda()).sum().backward()
    finally:
        ops.set_precision("tf32")
    e, ex = rel_err(y, ref), rel_err(xg.grad, xr.grad)
    print("bf16 mode, small stack: fwd %.2e dx %.2e" % (e, ex))
    assert e < 2e-2 and ex < 5e-2
