"""sx_gemm's transposed second output (`ct`): the epilogue writes every final value of C a second time, transposed.

`ct` holds the values after alpha, bias, activation, dropout and TF32 rounding, so it must equal C transposed bit for
bit, on both tile widths, at ragged shapes and with strided batch layouts.  The autograd node that reads such copies
(P.V' -> GELU -> grouped output Linear) must give the bits of the MN-major path with the K-major copies on and off.
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


def at_width(wide, fn):
    import segtran_b200._lib as L
    try:
        L.call("sx_gemm_debug_set", b"wide_tiles", 1 if wide else 0)
        out = fn()
        torch.cuda.synchronize()
    finally:
        L.call("sx_gemm_debug_set", b"wide_tiles", -1)
    return out


def ct_like(Z1, Z0, M, N, pad=4):
    """[Z1, Z0, N, M] view with the row pitch padded past M (a 16-byte multiple) and a gap between the z slices"""
    ld = (M + pad + 3) // 4 * 4
    buf = torch.full((Z1, Z0 * N + 3, ld), float("nan"), device="cuda")
    return buf[:, :Z0 * N].view(Z1, Z0, N, ld)[..., :M]


# (M, N, K, Z1, Z0): odd M and N against both tile widths, a partial last k-block, batches
SHAPES = [(301, 523, 200, 2, 3), (2743, 1001, 96, 1, 1), (130, 257, 40, 1, 2), (64, 40, 32, 1, 1)]


@pytest.mark.parametrize("wide", [0, 1], ids=["narrow", "wide"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_ct_is_c_transposed_for_every_epilogue(shape, wide):
    import segtran_b200._lib as L
    from segtran_b200 import ops
    M, N, K, Z1, Z0 = shape
    a = tf32(torch.randn(Z1, Z0, M, K, device="cuda"))
    b = tf32(torch.randn(Z1, Z0, N, K, device="cuda"))
    bias_n = torch.randn(N, device="cuda")
    bias_m = torch.randn(M, device="cuda")
    pre = torch.randn(Z1, Z0, M, N, device="cuda")
    kw = [dict(round_out=False), dict(alpha=0.37), dict(bias=bias_n), dict(bias=bias_m, bias_mode=L.SX_BIAS_M),
          dict(bias=bias_n, gelu=True, drop_p=0.25, seed=7), dict(gelu_bwd=pre, drop_p=0.2, seed=11),
          dict(drop_p=0.5, seed=3), dict(amax=True)]
    for k in kw:
        k = dict(k)
        amax = None
        if k.pop("amax", False):
            amax = k["amax"] = torch.full((1,), -3.0e38, device="cuda")
        h = torch.empty(Z1, Z0, M, N, device="cuda") if k.get("gelu") else None
        if h is not None:
            k["preact"] = h

        def run():
            ct = ct_like(Z1, Z0, M, N)
            c = ops.gemm_nt(a, b, split_k=1, ct=ct, **k)
            return c, ct

        c, ct = at_width(wide, run)
        ref = at_width(wide, lambda: ops.gemm_nt(a, b, split_k=1, **{**k, "amax": None} if amax is not None else k))
        assert torch.equal(c, ref), k                           # the second output leaves C unchanged
        assert torch.equal(ct, c.transpose(-1, -2)), k
        if h is not None:
            assert not torch.isnan(h).any()


def test_ct_with_broadcast_operands():
    from segtran_b200 import ops
    a = tf32(torch.randn(2, 3, 300, 200, device="cuda"))
    w = tf32(torch.randn(1, 1, 520, 200, device="cuda"))
    for wide in (0, 1):
        ct = ct_like(2, 3, 300, 520)
        c = at_width(wide, lambda: ops.gemm_nt(a, w, split_k=1, ct=ct))
        assert torch.equal(ct, c.transpose(-1, -2))


def test_invalid_combinations_are_refused():
    import segtran_b200._lib as L
    from segtran_b200 import ops
    a = tf32(torch.randn(1, 1, 256, 4096, device="cuda"))
    b = tf32(torch.randn(1, 1, 256, 4096, device="cuda"))
    ct = ct_like(1, 1, 256, 256)
    with pytest.raises(L.SxError, match="ct"):
        ops.gemm_nt(a, b, split_k=4, ct=ct)                     # split-K
    acc = torch.zeros(1, 1, 256, 256, device="cuda")
    with pytest.raises(L.SxError, match="ct"):
        ops.gemm_nt(a, b, out=acc, accumulate=True, split_k=1, ct=ct, round_out=False)
    with pytest.raises(L.SxError, match="ct"):                  # an MN-major operand
        ops.gemm_nt(a, b.transpose(-1, -2).contiguous().transpose(-1, -2), split_k=1, ct=ct)
    with pytest.raises(L.SxError, match="ct"):                  # a row pitch that is not a 16-byte multiple
        ops.gemm_nt(a, b, split_k=1, ct=torch.empty(256, 258, device="cuda")[:, :256])


def _pv_node(copies):
    from segtran_b200 import ops
    B, M, U1, U2, Fd = 2, 4, 1101, 512, 1024
    g = torch.Generator(device="cuda").manual_seed(1)
    P = tf32(torch.rand(B, M, U1, U2, device="cuda", generator=g) / U2).requires_grad_()
    v = tf32(torch.randn(B, U2, M * Fd, device="cuda", generator=g)).requires_grad_()
    bm = torch.randn(Fd, device="cuda", generator=g).requires_grad_()
    Wo = (torch.randn(M * Fd, Fd, 1, device="cuda", generator=g) / 32).requires_grad_()
    bo = torch.randn(M * Fd, device="cuda", generator=g).requires_grad_()
    dY = torch.randn(B, M, U1, Fd, device="cuda", generator=g)
    ops.set_kmajor_copies(copies)
    try:
        assert ops._token_kmajor(Fd, Fd, U1, M) == copies and ops._token_kmajor(U2, Fd, U1, B * M) == copies
        Y = ops.attn_pv_gelu_group_linear(P, v, M, bm, 0.2, 5, Wo, bo)
        Y.backward(dY)
        torch.cuda.synchronize()
    finally:
        ops.set_kmajor_copies(True)
    return [Y.detach()] + [t.grad for t in (P, v, bm, Wo, bo)]


def test_pv_gelu_group_linear_node_copies_on_and_off():
    on, off = _pv_node(True), _pv_node(False)
    for i, (x, y) in enumerate(zip(on, off)):
        assert torch.equal(x, y), (i, float((x - y).abs().max()))


def _pv_plain(copies):
    """the in-squeeze form P1 h (one mode, attractor rows against token keys): forward and both gradients"""
    from segtran_b200 import ops
    B, A, N, C = 4, 1024, 1100, 1024
    g = torch.Generator(device="cuda").manual_seed(2)
    P = tf32(torch.rand(B, 1, A, N, device="cuda", generator=g) / N).requires_grad_()
    h = tf32(torch.randn(B, N, C, device="cuda", generator=g)).requires_grad_()
    dU = torch.randn(B, 1, A, C, device="cuda", generator=g)
    ops.set_kmajor_copies(copies)
    try:
        assert ops._token_kmajor(A, C, N, B) == copies and ops._token_kmajor(N, C, A, B) == copies
        U = ops.attn_pv(P, h, 1)
        U.backward(dU)
        torch.cuda.synchronize()
    finally:
        ops.set_kmajor_copies(True)
    return [U.detach(), P.grad, h.grad]


def test_attn_pv_node_copies_on_and_off():
    on, off = _pv_plain(True), _pv_plain(False)
    for i, (x, y) in enumerate(zip(on, off)):
        assert torch.equal(x, y), (i, float((x - y).abs().max()))


def test_ct_is_written_only_by_the_call_given_it():
    """a refused call leaves ct untouched, and a call without ct never writes it, before or after one with it"""
    import segtran_b200._lib as L
    from segtran_b200 import ops
    a = tf32(torch.randn(1, 1, 256, 512, device="cuda"))
    b = tf32(torch.randn(1, 1, 256, 512, device="cuda"))
    ct = ct_like(1, 1, 256, 256)
    acc = torch.zeros(1, 1, 256, 256, device="cuda")
    with pytest.raises(L.SxError, match="ct"):
        ops.gemm_nt(a, b, out=acc, accumulate=True, split_k=1, ct=ct, round_out=False)
    ops.gemm_nt(a, b, split_k=1)
    torch.cuda.synchronize()
    assert torch.isnan(ct).all()
    c = ops.gemm_nt(a, b, split_k=1, ct=ct)
    assert torch.equal(ct, c.transpose(-1, -2))
    ct.fill_(float("nan"))
    ops.gemm_nt(b, a, split_k=1)
    torch.cuda.synchronize()
    assert torch.isnan(ct).all()
