"""sx_gemm's 128 x 256 tiles (TF32, both operands K-major) against its 128 x 128 tiles: bit-identical outputs.

The wide tile changes only how many output columns one CTA owns.  Every output element still sees the same k-blocks
in the same order and the same k8 MMA steps, and the epilogue runs the same per-element arithmetic, so forcing the
wide tile must give exactly the bits of the narrow one for every epilogue, ragged shape and batch layout.
"""

import pytest
import torch

pytestmark = pytest.mark.gpu


def tf32(x):
    u = x.contiguous().view(torch.int32)
    u = (u + 0x0FFF + ((u >> 13) & 1)) & ~0x1FFF
    return u.view(torch.float32)


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)


def both_widths(fn):
    """fn() with the wide tile forced off, then forced on (wherever legal)"""
    import segtran_b200._lib as L
    try:
        L.call("sx_gemm_debug_set", b"wide_tiles", 0)
        narrow = fn()
        torch.cuda.synchronize()
        L.call("sx_gemm_debug_set", b"wide_tiles", 1)
        wide = fn()
        torch.cuda.synchronize()
    finally:
        L.call("sx_gemm_debug_set", b"wide_tiles", -1)
    return narrow, wide


def assert_same(narrow, wide):
    if isinstance(narrow, torch.Tensor):
        narrow, wide = (narrow,), (wide,)
    for i, (n, w) in enumerate(zip(narrow, wide)):
        assert torch.equal(n, w), (i, float((n - w).abs().max()))


# (M, N, K, Z1, Z0): ragged M and N against both tile widths, a partial last k-block, batches
SHAPES = [(300, 520, 200, 2, 3), (2744, 1000, 96, 1, 1), (2744, 136, 64, 1, 2), (130, 257, 40, 1, 1)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_plain_and_rounded(shape):
    from segtran_b200 import ops
    M, N, K, Z1, Z0 = shape
    a = tf32(torch.randn(Z1, Z0, M, K, device="cuda"))
    b = tf32(torch.randn(Z1, Z0, N, K, device="cuda"))
    assert_same(*both_widths(lambda: (ops.gemm_nt(a, b, split_k=1, round_out=False),
                                      ops.gemm_nt(a, b, alpha=0.37, split_k=1, round_out=True))))


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_epilogues(shape):
    import segtran_b200._lib as L
    from segtran_b200 import ops
    M, N, K, Z1, Z0 = shape
    a = tf32(torch.randn(Z1, Z0, M, K, device="cuda"))
    b = tf32(torch.randn(Z1, Z0, N, K, device="cuda"))
    bias_n = torch.randn(N, device="cuda")
    bias_m = torch.randn(M, device="cuda")
    addend = torch.randn(Z1, Z0, M, N, device="cuda")
    pre = torch.randn(Z1, Z0, M, N, device="cuda")

    def run():
        h = torch.empty(Z1, Z0, M, N, device="cuda")
        amax = torch.full((1,), -3.0e38, device="cuda")
        acc = torch.ones(Z1, Z0, M, N, device="cuda")
        return (ops.gemm_nt(a, b, bias=bias_n, split_k=1),
                ops.gemm_nt(a, b, bias=bias_m, bias_mode=L.SX_BIAS_M, split_k=1),
                ops.gemm_nt(a, b, addend=addend, split_k=1),
                ops.gemm_nt(a, b, bias=bias_n, gelu=True, preact=h, drop_p=0.25, seed=7, split_k=1), h,
                ops.gemm_nt(a, b, gelu_bwd=pre, drop_p=0.2, seed=11, split_k=1, round_out=False),
                ops.gemm_nt(a, b, drop_p=0.5, seed=3, split_k=1),
                ops.gemm_nt(a, b, amax=amax, split_k=1, round_out=True), amax,
                ops.gemm_nt(a, b, out=acc, accumulate=True, split_k=1, round_out=False))

    assert_same(*both_widths(run))


def test_broadcast_operands_and_z1_fold():
    from segtran_b200 import ops
    a = tf32(torch.randn(2, 3, 300, 200, device="cuda"))
    b = tf32(torch.randn(2, 3, 520, 200, device="cuda"))
    w = tf32(torch.randn(1, 1, 520, 200, device="cuda"))        # stride-0 over both batch dims
    w1 = tf32(torch.randn(2, 1, 520, 200, device="cuda"))       # stride-0 over z0 only
    x = tf32(torch.randn(1, 3, 300, 200, device="cuda"))        # A broadcast over z1
    assert_same(*both_widths(lambda: (ops.gemm_nt(a, w, split_k=1, round_out=False),
                                      ops.gemm_nt(a, w1, split_k=1, round_out=False),
                                      ops.gemm_nt(x, b, split_k=1, round_out=False),
                                      ops.gemm_nt(a, b, reduce_z1=True, split_k=1, round_out=False),
                                      ops.gemm_nt(x, b, reduce_z1=True, split_k=1, round_out=False))))


def test_grid_size_on_wide_tiles():
    """a few CTAs that each walk many wide tiles give the bits of one tile per CTA"""
    import segtran_b200._lib as L
    from segtran_b200 import ops
    a = tf32(torch.randn(2, 3, 296, 200, device="cuda"))
    b = tf32(torch.randn(2, 3, 520, 200, device="cuda"))
    bias = torch.randn(520, device="cuda")
    try:
        L.call("sx_gemm_debug_set", b"wide_tiles", 1)
        ref = ops.gemm_nt(a, b, bias=bias, gelu=True, drop_p=0.25, seed=99, split_k=1)
        for ctas in (7, 1):
            L.call("sx_gemm_debug_set", b"max_ctas", ctas)
            assert torch.equal(ops.gemm_nt(a, b, bias=bias, gelu=True, drop_p=0.25, seed=99, split_k=1), ref), ctas
    finally:
        L.call("sx_gemm_debug_set", b"max_ctas", -1)
        L.call("sx_gemm_debug_set", b"wide_tiles", -1)


def test_wide_tile_against_fp64():
    """the wide tile at a ragged shape against an fp64 product of the same TF32 operands"""
    import segtran_b200._lib as L
    from segtran_b200 import ops
    a = tf32(torch.randn(2, 650, 300, device="cuda"))
    b = tf32(torch.randn(2, 1000, 300, device="cuda"))
    bias = torch.randn(1000, device="cuda")
    try:
        L.call("sx_gemm_debug_set", b"wide_tiles", 1)
        got = ops.gemm_nt(a, b, bias=bias, alpha=0.5, split_k=1, round_out=False)
    finally:
        L.call("sx_gemm_debug_set", b"wide_tiles", -1)
    ref = 0.5 * (a.double() @ b.double().transpose(-1, -2)) + bias.double()
    err = float((got.view_as(ref).double() - ref).abs().max() / ref.abs().max())
    assert err < 1e-5, err
