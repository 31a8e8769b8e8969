"""sx_gemm bit-exactness across operand majorness and persistent-grid sizes.

TF32 wgmma reads K-major shared memory only, so an MN-major TF32 operand is rewritten into the K-major layout inside
the kernel before its MMAs.  That rewrite must be exact: the K-major and MN-major views of the same values give the
same bits.  The tile schedule must not change any output either: a grid of a few CTAs that each walk many tiles (and
carry the operand rings and barrier phases across them) gives the same bits as one tile per CTA.
"""

import pytest
import torch

pytestmark = pytest.mark.gpu


def tf32(x):
    u = x.contiguous().view(torch.int32)
    u = (u + 0x0FFF + ((u >> 13) & 1)) & ~0x1FFF
    return u.view(torch.float32)


def mn_major(x):
    """the same values with the second-to-last dim contiguous"""
    return x.transpose(-1, -2).contiguous().transpose(-1, -2)


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)


def test_gemm_majorness_is_bit_exact():
    from segtran_b200 import ops
    # ragged M / N / K (partial tiles and a partial last k-block), batched, several k-blocks per tile
    a = tf32(torch.randn(2, 3, 300, 200, device="cuda"))
    b = tf32(torch.randn(2, 3, 520, 200, device="cuda"))
    bias = torch.randn(520, device="cuda")
    ref = ops.gemm_nt(a, b, split_k=1, round_out=False)
    ref_epi = ops.gemm_nt(a, b, bias=bias, gelu=True, drop_p=0.25, seed=7)
    for x, y in ((a, mn_major(b)), (mn_major(a), b), (mn_major(a), mn_major(b))):
        assert torch.equal(ops.gemm_nt(x, y, split_k=1, round_out=False), ref)
        assert torch.equal(ops.gemm_nt(x, y, bias=bias, gelu=True, drop_p=0.25, seed=7), ref_epi)
    # split-K and batch-reduced launches sum their partials in a fixed order: also bit-exact across majorness
    red = ops.gemm_nt(a, b, reduce_z1=True, round_out=False)
    sk = ops.gemm_nt(a, b, split_k=3, round_out=False)
    for x, y in ((a, mn_major(b)), (mn_major(a), mn_major(b))):
        assert torch.equal(ops.gemm_nt(x, y, reduce_z1=True, round_out=False), red)
        assert torch.equal(ops.gemm_nt(x, y, split_k=3, round_out=False), sk)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_gemm_grid_size_is_bit_exact(precision):
    import segtran_b200._lib as L
    from segtran_b200 import ops
    # MN-major operands need 16-byte pitches, also in bf16: 296 rows (ragged against the 128-row tiles)
    a = tf32(torch.randn(2, 3, 296, 200, device="cuda"))
    b = tf32(torch.randn(2, 3, 520, 200, device="cuda"))
    am, bm = mn_major(a), mn_major(b)
    bias = torch.randn(520, device="cuda")

    def run():
        h = torch.empty(2, 3, 296, 520, device="cuda")
        return (ops.gemm_nt(a, bm, bias=bias, gelu=True, preact=h, drop_p=0.25, seed=99), h,
                ops.gemm_nt(am, bm, split_k=1, round_out=False),
                ops.gemm_nt(am, bm, reduce_z1=True, round_out=False),
                ops.gemm_nt(am, b[:1, :1], split_k=3, accumulate=True, out=torch.ones(2, 3, 296, 520, device="cuda"),
                            round_out=False))

    ops.set_precision(precision)
    try:
        ref = run()
        for ctas in (7, 2, 1):
            L.call("sx_gemm_debug_set", b"max_ctas", ctas)
            got = run()
            for i, (g, r) in enumerate(zip(got, ref)):
                assert torch.equal(g, r), (ctas, i)
    finally:
        L.call("sx_gemm_debug_set", b"max_ctas", -1)
        ops.set_precision("tf32")
