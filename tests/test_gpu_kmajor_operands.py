"""K-major copies of the small MN-major operands of single-pass TF32 products (ops.set_kmajor_copies).

TF32 wgmma reads only K-major shared memory, so sx_gemm rewrites an MN-major TF32 operand before its MMAs and such a
launch runs at about half the K-major rate.  The training step therefore hands the weight-, key- and value-bank-side
operands over as transposed copies.  These tests check, on one training step of the cfg-4 stack (Segtran3d BraTS 112^3,
batch 1 instead of 4: majorness does not depend on the batch), that
  (a) every single-pass TF32 launch that still reads an MN-major operand is one of the token contractions whose operands
      are both large (weight gradients, dV' = P^T dH, dK = dS^T Q, the in-squeeze products, the head's convolutions,
      the weight-space value-bank fold), and the two launches that made the step slow are gone;
  (b) the step computes the same bits with the copies on and off.
"""
import math
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

# call-site text of the products allowed to keep an MN-major operand, and why
INHERENT = {
    "dy2.t(), x2.t()": "Linear weight gradient dY^T X (token rows)",
    "dY.transpose(-1, -2), G.transpose(-1, -2)": "grouped output Linear weight gradient dY^T G (token rows)",
    "dS.transpose(-1, -2), _head_cols(q,": "dK = dS^T Q (token contraction)",
    "gemm_nt(dS, _head_cols(k,": "in-squeeze dQ = dS K with the token keys",
    "gemm_nt(P, vv,": "in-squeeze P1 h with the token values",
    "gemm_nt(dU, v.view": "in-squeeze backward dP1 = dU h^T",
    "P.transpose(-1, -2), dU.transpose(-1, -2)": "dV' = P^T dH and the in-squeeze backward dh = P1^T dU (token contractions)",
    "Wvr.transpose(-1, -2)": "weight-space value-bank fold W' = Wm Wv",
    "d2.t(), a2.t()": "value-bank fold weight gradient (attractor rows)",
    "Wmr.t().view(1, 1, Fd, Fd)": "value-bank fold backward, weight space",
    "xr.view(B, 1, Cin, V).transpose(-1, -2)": "1x1 convolution on a channels-first activation",
    "dy.view(B, 1, Cout, V).transpose(-1, -2)": "1x1 convolution backward on a channels-first gradient",
    "vf.transpose(1, 2).unsqueeze(1)": "head class-conv weight gradient dWc (token contraction)",
}


def _call_text(frame):
    """Source text of the call the frame is executing (all lines of a multi-line call)."""
    import linecache
    code = frame.f_code
    pos = list(code.co_positions())[frame.f_lasti // 2]
    lo, hi = pos[0], pos[1] or pos[0]
    return " ".join(linecache.getline(code.co_filename, i).strip() for i in range(lo, hi + 1))


class _GemmRecorder:
    def __init__(self):
        self.launches = []                  # (shape label, op dtype, A major, B major, caller qualname, call text)

    def __call__(self, name, cargs):
        import contextlib
        if name == "sx_gemm":
            g = cargs[0]._obj
            f = sys._getframe(1)
            while f is not None and (not f.f_code.co_filename.endswith("ops.py") or
                                     f.f_code.co_name in ("gemm_nt", "_gemm_nt_1", "_param_grad", "call")):
                f = f.f_back
            site = (f.f_code.co_qualname, _call_text(f)) if f is not None else ("?", "?")
            self.launches.append(("%dx%dx%d z%d" % (g.M, g.N, g.K, g.Z0 * g.Z1), g.op_dtype, g.A.major, g.B.major) + site)
        return contextlib.nullcontext()


def _cfg4_step(B=1, dropout=0.2):
    import bench
    from segtran_b200.train import seg_loss
    c = bench.CONFIGS[4]
    net = bench.build_net(c, "cuda", dropout=dropout).cuda().train()
    hp = bench.hot_params(net, c)
    feat, curr, Y = bench.synthetic_batch(c, B, torch.device("cuda"), 4242)
    pw, cw = bench.loss_weights(c, "cuda")
    sp = (c["S"],) * 3

    def step():
        for p in hp:
            p.grad = None
        f = feat.clone().requires_grad_()
        cc = curr.clone().requires_grad_()
        logits = net.hot_path(f, cc, None, sp)
        loss, _, _ = seg_loss(logits, Y.float(), pw, cw, bench.TRAIN["dice_w"])
        loss.backward()
        return [loss.detach(), logits.detach(), f.grad, cc.grad] + [p.grad for p in hp]

    return step


@pytest.fixture(autouse=True)
def _restore():
    from segtran_b200 import _lib as L
    from segtran_b200 import ops
    yield
    L.set_hook(None)
    ops.set_kmajor_copies(True)
    ops.set_precision("tf32")


def test_cfg4_step_reads_mn_major_tf32_operands_only_in_token_contractions_and_squeeze_out_dq_copies_keys():
    from segtran_b200 import _lib as L
    from segtran_b200 import ops
    ops.set_kmajor_copies(True)
    step = _cfg4_step()
    rec = _GemmRecorder()
    L.set_hook(rec)
    step()
    torch.cuda.synchronize()
    L.set_hook(None)
    tf32 = [x for x in rec.launches if x[1] == L.SX_OP_TF32]
    assert len(tf32) > 20
    mn = [x for x in tf32 if x[2] == L.SX_MAJOR_MN or x[3] == L.SX_MAJOR_MN]
    bad = [x for x in mn if not any(s in x[5] for s in INHERENT)]
    assert not bad, "single-pass TF32 launches with an MN-major operand outside the token contractions:\n" + \
        "\n".join(map(str, bad))
    # the squeeze-out's P.V' and dH = dY Wo ([B*modes] x 2744 x 1024 x 1024) now read both operands K-major
    big = [x for x in tf32 if x[0] == "2744x1024x1024 z4"]
    assert len(big) >= 4 and all(x[2] == x[3] == L.SX_MAJOR_K for x in big), big
    # the squeeze-out's dQ = dS K (tokens x key width x attractors, one batch per mode) shares its call site with the
    # in-squeeze dQ, which reads the token keys MN-major; it reads a K-major copy of the attractor keys
    import bench
    c = bench.CONFIGS[4]
    dq = [x for x in tf32 if x[0] == "%dx%dx%d z%d" % (math.prod(c["grid"]), c["dims"][0] // c["modes"], c["attractors"],
                                                        c["modes"])]
    assert dq and all(x[2] == x[3] == L.SX_MAJOR_K for x in dq), dq


def test_cfg4_step_is_bit_identical_with_and_without_kmajor_copies():
    from segtran_b200 import ops
    step = _cfg4_step()
    step()                                          # creates the device base seed, so reseed() below pins it
    outs = []
    for on in (False, True, False):
        ops.set_kmajor_copies(on)
        ops.reseed(1234)
        ops._site_counter[0] = 0
        outs.append([None if t is None else t.clone() for t in step()])   # (parameters outside the graph: None)
        torch.cuda.synchronize()
    names = ["loss", "logits", "feat_grad", "curr_grad"]
    for i, (a, b, c) in enumerate(zip(*outs)):
        name = names[i] if i < len(names) else "param_grad[%d]" % (i - len(names))
        if a is None:
            assert b is None and c is None, name
            continue
        assert torch.equal(a, c), "the step is not reproducible: " + name
        assert torch.equal(a, b), name


@pytest.mark.parametrize("Z,R,C", [(3, 13, 7), (2, 12, 8), (1, 301, 40), (4, 16, 128), (2, 1024, 36)])
def test_transposed_copy_has_padded_rows_and_exact_values(Z, R, C):
    """sx_transpose with an output row pitch: the vectorised path (R, C multiples of 4) and the scalar one."""
    from segtran_b200 import ops
    torch.manual_seed(1)
    x = torch.randn(Z, R, C, device="cuda")
    y = ops._transposed(x, Z, R, C)
    assert y.shape == (Z, C, R) and y.stride() == (C * ((R + 3) // 4 * 4), (R + 3) // 4 * 4, 1)
    assert torch.equal(y, x.transpose(1, 2))


@pytest.mark.parametrize("fused,U2", [(True, 300), (False, 300), (False, 301)])
def test_squeeze_out_is_bit_identical_with_and_without_kmajor_copies(fused, U2):
    """Ragged shapes (partial tiles; 301 keys: padded copy rows), both dropouts, the fused and the separate-kernel
    squeeze-out."""
    from segtran_b200 import ops
    from tests.test_gpu_attn import _fused, _sq_inputs, _unfused
    B, M, U1, d, Fd = 2, 2, 260, 32, 64
    res = []
    for on in (False, True):
        ops.set_kmajor_copies(on)
        q, k, vp, bm, Wo, bo, gY = _sq_inputs(B, M, U1, U2, d, Fd, seed=5)
        if fused:
            diag = torch.tensor([-3.0e38, 0.0, 0.0], device="cuda")
            Y = _fused(q, k, vp, M, 0.2, 1111, bm, 0.2, 2222, Wo, bo, diag)
        else:
            Y = _unfused(q, k, vp, M, 0.2, 1111, bm, 0.2, 2222, Wo, bo)
        (Y * gY).sum().backward()
        res.append([Y.detach()] + [t.grad for t in (q, k, vp, bm, Wo, bo)])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_linear_input_gradient_with_and_without_kmajor_copies_is_bit_identical():
    """Ragged shapes: 210 token rows, 36 outputs, 52 inputs (partial tiles in every dimension)."""
    from segtran_b200 import ops
    torch.manual_seed(2)
    x = torch.randn(3, 70, 52, device="cuda")
    W = torch.randn(36, 52, device="cuda") * 0.1
    b = torch.randn(36, device="cuda")
    gy = torch.randn(3, 70, 36, device="cuda")
    res = []
    for on in (False, True):
        ops.set_kmajor_copies(on)
        xl, Wl = x.clone().requires_grad_(), W.clone().requires_grad_()
        (ops.linear(xl, Wl, b, gelu=True) * gy).sum().backward()
        res.append((xl.grad, Wl.grad))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
