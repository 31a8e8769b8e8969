"""Transposed probabilities from the attention kernel, and K-major operands for the step's weight-gradient and in-squeeze
products.

  (a) sx_attn_probs_fwd's optional P^T output holds exactly the transpose of P (biased and unbiased, with and without
      dropout, one- and two-pass key counts, query counts that are not a multiple of the 128-row block), and asking for
      it leaves P, lse and the statistics unchanged;
  (b) on one training step of the cfg-4 stack at its batch of 4, dV' = P^T dH reads the kernel's P^T (no transpose pass
      over P); the tokens are transposed once per layer, and P1 h, d(Q1 Wk) = dS1 h and the squeeze-out query
      projection's dWq = dQ^T h read that copy; and dWq, the folded value bank's dW' = dV'^T a and dWv = Wm^T dW',
      and the in-squeeze's dh = dS1^T (Q1 Wk) read both operands K-major;
  (c) that step computes the same bits with the K-major operands on and off.
"""
import sys

import pytest
import torch

from tests.test_gpu_kmajor_operands import _cfg4_step

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore():
    from segtran_b200 import _lib as L
    from segtran_b200 import ops
    yield
    L.set_hook(None)
    ops.set_kmajor_copies(True)
    ops.set_precision("tf32")


def _qk(B, Bq, M, U1, U2, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(Bq, U1, M * d, device="cuda", generator=g)
    k = torch.randn(B, U2, M * d, device="cuda", generator=g)
    return q, k


@pytest.mark.parametrize("B,Bq,M,U1,U2,d", [(2, 2, 2, 260, 100, 32), (2, 2, 2, 260, 300, 32), (3, 1, 1, 130, 257, 64),
                                            (1, 1, 4, 128, 128, 16)])
@pytest.mark.parametrize("drop_p", [0.0, 0.2])
def test_transposed_probs_equal_p_transposed(B, Bq, M, U1, U2, d, drop_p):
    from segtran_b200 import ops
    q, k = _qk(B, Bq, M, U1, U2, d, seed=U1 + U2)
    ref = ops.attn_probs_fused(q, k, M, drop_p=drop_p, seed=77, need_scores=True)
    Pt = ops._rowpad_empty((B, M, U2, U1), q.device)
    out = ops.attn_probs_fused(q, k, M, drop_p=drop_p, seed=77, need_scores=True, pt=Pt)
    for a, b in zip(ref, out):
        assert torch.equal(a, b)
    assert torch.equal(Pt, out[0].transpose(-1, -2))


@pytest.mark.parametrize("grid,R", [((5, 5, 5), 2), ((6, 6, 6), 3), ((13, 11), 4)])
@pytest.mark.parametrize("drop_p", [0.0, 0.2])
def test_transposed_probs_with_positional_biases(grid, R, drop_p):
    """125 tokens: one pass; 216 and 143 tokens: two passes and a partial row block."""
    from segtran_b200 import ops
    N = 1
    for g in grid:
        N *= g
    B, M, d = 2, 2, 32
    q, k = _qk(B, B, M, N, N, d, seed=N)
    table = torch.randn((2 * R + 1,) * len(grid), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    pb = ops.PosBias(table, R, grid, 0.7)
    ref = ops.attn_probs_fused(q, k, M, drop_p=drop_p, seed=5, need_scores=True, posbias=pb)
    Pt = ops._rowpad_empty((B, M, N, N), q.device)
    out = ops.attn_probs_fused(q, k, M, drop_p=drop_p, seed=5, need_scores=True, posbias=pb, pt=Pt)
    for a, b in zip(ref, out):
        assert torch.equal(a, b)
    assert torch.equal(Pt, out[0].transpose(-1, -2))


class _Recorder:
    def __init__(self):
        self.gemms = []           # (shape label, A major, B major, caller qualname)
        self.transposes = []      # (Z, R, C, caller qualname)
        self.attn_pt = []         # one flag per sx_attn_probs_fwd call: P^T requested

    def __call__(self, name, cargs):
        import contextlib
        f = sys._getframe(1)
        while f is not None and (not f.f_code.co_filename.endswith("ops.py") or
                                 f.f_code.co_name in ("gemm_nt", "_gemm_nt_1", "_param_grad", "call", "_transposed",
                                                      "_head_cols")):
            f = f.f_back
        site = f.f_code.co_qualname if f is not None else "?"
        if name == "sx_gemm":
            g = cargs[0]._obj
            self.gemms.append(("%dx%dx%d z%d" % (g.M, g.N, g.K, g.Z0 * g.Z1), g.A.major, g.B.major, site))
        elif name == "sx_transpose":
            self.transposes.append((cargs[1], cargs[2], cargs[3], site))
        elif name == "sx_attn_probs_fwd":
            self.attn_pt.append(cargs[1] is not None)
        return contextlib.nullcontext()


def test_cfg4_step_reads_transposed_probs_and_kmajor_weight_gradient_and_in_squeeze_operands():
    import bench
    from segtran_b200 import _lib as L
    from segtran_b200 import ops
    ops.set_kmajor_copies(True)
    c = bench.CONFIGS[4]
    B, N, A, C, M = c["B"], 1, c["attractors"], c["dims"][0], c["modes"]    # C: token width = each mode's value width
    for g in c["grid"]:
        N *= g
    step = _cfg4_step(B=B)
    rec = _Recorder()
    L.set_hook(rec)
    step()
    torch.cuda.synchronize()
    L.set_hook(None)
    K = L.SX_MAJOR_K

    def launches(shape, site):
        return [x for x in rec.gemms if x[0] == shape and x[3] == site]

    # the squeeze-out's attention kernel writes P^T, and nothing transposes P [B*M, N, A] any more
    assert rec.attn_pt and all(rec.attn_pt), rec.attn_pt
    assert not [t for t in rec.transposes if t == (B * M, N, A, "_pv_grads")], rec.transposes
    dv = launches("%dx%dx%d z%d" % (A, C, N, B * M), "_pv_grads")
    assert dv and all(x[1] == x[2] == K for x in dv), dv
    # folded value bank: dW' = dV'^T a over the B*A bank rows
    dwf = launches("%dx%dx%d z1" % (M * C, C, B * A), "_FoldedValueBank.backward")
    assert dwf and all(x[1] == x[2] == K for x in dwf), rec.gemms
    # ... and its weight-space products dWm = sum_m dW'_m Wv_m and dWv_m = Wm^T dW'_m (dW'^T from that product's `ct`)
    dwv = launches("%dx%dx%d z%d" % (C, C, C, M), "_FoldedValueBank.backward")
    assert len(dwv) == 2 and all(x[1] == x[2] == K for x in dwv), dwv
    # the tokens [B, N, C] are transposed once, as one [B*N, C] matrix, not per sample for the in-squeeze products
    assert [t for t in rec.transposes if t == (1, B * N, C, "tokens_t")], rec.transposes
    assert not [t for t in rec.transposes if t[:3] == (B, N, C) and t[3] in ("_AttnPV.forward", "_score_grads")], \
        rec.transposes
    dwq = launches("%dx%dx%d z1" % (C, C, B * N), "_Linear.backward")
    assert dwq and all(x[1] == x[2] == K for x in dwq), dwq
    # in-squeeze (one mode over the N tokens): P1 h, d(Q1 Wk) = sum_b dS1 h and dh = dS1^T (Q1 Wk)
    p1h = launches("%dx%dx%d z%d" % (A, C, N, B), "_AttnPV.forward")
    assert p1h and all(x[1] == x[2] == K for x in p1h), p1h
    dq = launches("%dx%dx%d z%d" % (A, C, N, B), "_score_grads")
    dk = launches("%dx%dx%d z%d" % (N, C, A, B), "_score_grads")
    assert dq and all(x[1] == x[2] == K for x in dq), dq
    assert dk and all(x[1] == x[2] == K for x in dk), dk


def test_cfg4_step_at_batch_4_is_bit_identical_with_and_without_kmajor_operands():
    from segtran_b200 import ops
    step = _cfg4_step(B=4)
    step()                                          # creates the device base seed, so reseed() below pins it
    outs = []
    for on in (True, False):
        ops.set_kmajor_copies(on)
        ops.reseed(1234)
        ops._site_counter[0] = 0
        outs.append([None if t is None else t.clone() for t in step()])
        torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(*outs)):
        if a is None:
            assert b is None, i
            continue
        assert torch.equal(a, b), i
