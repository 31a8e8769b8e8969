"""Time the step's token-contracted TF32 products three ways on the GPU (CUDA events, median of rounds):

  mn    both operands read MN-major in place (sx_gemm transposes them in shared memory, 128 x 128 tiles)
  copy  both operands transposed first by sx_transpose (read + write), then a K-major product (128 x 256 tiles)
  ct    one operand comes transposed out of the epilogue of the GEMM that makes it (counted: that GEMM with and
        without `ct`), the other through sx_transpose, then the K-major product
  Pt    dV' = P^T dH with P^T written by the attention kernel (counted: sx_attn_probs_fwd with and without it) and dH^T
        by its producer's `ct`: the K-major product alone

and the weight-gradient and in-squeeze products that read K-major copies where ops._token_kmajor takes them: the folded
value bank's dW' = dV'^T a (bank rows B*A), the in-squeeze's d(Q1 Wk) = sum_b dS1 h and dh = dS1^T (Q1 Wk) (one mode over
the tokens), each mn and copy, and the squeeze-out query projection's dWq = dQ^T h over the B*N token rows (split 2): mn,
and twin (h^T is the layer's ops.tokens_t() copy, made anyway for P1 h; dQ through sx_transpose).

  python tools/time_token_contractions.py [--rounds 7] [--reps 10]

Shapes are cfg 4's (B = 4, 2744 tokens, 1024 attractors, 4 modes of 1024 channels).
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def tf32(x):
    u = x.contiguous().view(torch.int32)
    u = (u + 0x0FFF + ((u >> 13) & 1)) & ~0x1FFF
    return u.view(torch.float32)


def timed(fn, rounds, reps):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / reps)
    return statistics.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from segtran_b200 import ops
    assert torch.cuda.is_available(), "needs a GPU"
    B, M, U1, U2, Fd = 4, 4, 2744, 1024, 1024
    # dV' = P^T dH (z = B*M) and dWo = sum_b dY^T G (z0 = M, batch reduced): operands [B, M, tokens, 1024]
    P = tf32(torch.rand(B, M, U1, U2, device="cuda") / U2)
    dH = tf32(torch.randn(B, M, U1, Fd, device="cuda"))
    W = tf32(torch.randn(1, M, Fd, Fd, device="cuda"))             # the producer of dH: dY . Wo (K-major)
    dY = tf32(torch.randn(B, M, U1, Fd, device="cuda"))
    out = torch.empty(B, M, U2, Fd, device="cuda")
    acc = torch.zeros(1, M, Fd, Fd, device="cuda")
    ct = ops._rowpad_empty((B, M, Fd, U1), "cuda")
    dHt = ops._transposed(dH, B * M, U1, Fd).unflatten(0, (B, M))
    Pt = ops._transposed(P, B * M, U1, U2).unflatten(0, (B, M))
    # the squeeze-out's attention probabilities (queries = tokens, keys = attractors, 4 modes of 256)
    q = tf32(torch.randn(B, U1, Fd, device="cuda"))
    k = tf32(torch.randn(B, U2, Fd, device="cuda"))
    Pt_out = ops._rowpad_empty((B, M, U2, U1), "cuda")
    # folded value bank dW' = dV'^T a: dV' [B*A, M*F], a [B*A, C]
    dV = tf32(torch.randn(B * U2, M * Fd, device="cuda"))
    a = tf32(torch.randn(B * U2, Fd, device="cuda"))
    # in-squeeze, one mode: dS1 [B,1,A,N], h [B,N,C], Q1 Wk [1,A,C]
    dS1 = tf32(torch.randn(B, 1, U2, U1, device="cuda"))
    h = tf32(torch.randn(B, U1, Fd, device="cuda"))
    qw = tf32(torch.randn(1, U2, Fd, device="cuda"))
    dqw = torch.zeros(1, 1, U2, Fd, device="cuda")
    dh = torch.empty(B, 1, U1, Fd, device="cuda")
    # squeeze-out query projection: dQ [B*N, C], h^T [C, B*N]
    dQ = tf32(torch.randn(B * U1, Fd, device="cuda"))
    ht = ops._transposed(h, 1, B * U1, Fd)[0]
    gf = 2.0 * U2 * Fd * U1 * B * M / 1e9
    rows = []
    for name, fn in [
            ("P^T dH     mn  ", lambda: ops.gemm_nt(P.transpose(-1, -2), dH.transpose(-1, -2), out=out, round_out=False)),
            ("P^T dH     copy", lambda: ops.gemm_nt(ops._transposed(P, B * M, U1, U2).unflatten(0, (B, M)),
                                                     ops._transposed(dH, B * M, U1, Fd).unflatten(0, (B, M)), out=out,
                                                     round_out=False)),
            ("P^T dH     ct  ", lambda: ops.gemm_nt(ops._transposed(P, B * M, U1, U2).unflatten(0, (B, M)), dHt, out=out,
                                                     round_out=False)),
            ("P^T dH     Pt  ", lambda: ops.gemm_nt(Pt, dHt, out=out, round_out=False)),
            ("attn probs -   ", lambda: ops.attn_probs_fused(q, k, M, drop_p=0.2, seed=7, need_scores=True)),
            ("attn probs +Pt ", lambda: ops.attn_probs_fused(q, k, M, drop_p=0.2, seed=7, need_scores=True, pt=Pt_out)),
            ("dV'^T a    mn  ", lambda: ops.gemm_nt(dV.t(), a.t(), round_out=False)),
            ("dV'^T a    copy", lambda: ops.gemm_nt(ops._transposed(dV, 1, B * U2, M * Fd)[0],
                                                     ops._transposed(a, 1, B * U2, Fd)[0], round_out=False)),
            ("dS1 h      mn  ", lambda: ops.gemm_nt(dS1, h.view(B, 1, U1, Fd).transpose(-1, -2), out=dqw, reduce_z1=True,
                                                     split_k=1, round_out=False)),
            ("dS1 h      copy", lambda: ops.gemm_nt(dS1, ops._transposed(h, B, U1, Fd).unsqueeze(1), out=dqw,
                                                     reduce_z1=True, split_k=1, round_out=False)),
            ("dQ^T h     mn  ", lambda: ops.gemm_nt(dQ.t(), h.view(B * U1, Fd).t(), round_out=False)),
            ("dQ^T h     twin", lambda: ops.gemm_nt(ops._transposed(dQ, 1, B * U1, Fd)[0], ht, round_out=False)),
            ("dS1^T Q1Wk mn  ", lambda: ops.gemm_nt(dS1.transpose(-1, -2), qw.view(1, 1, U2, Fd).transpose(-1, -2),
                                                     out=dh, round_out=False)),
            ("dS1^T Q1Wk copy", lambda: ops.gemm_nt(ops._transposed(dS1, B, U2, U1).unsqueeze(1),
                                                     ops._transposed(qw, 1, U2, Fd).unsqueeze(1), out=dh,
                                                     round_out=False)),
            ("dY^T G     mn  ", lambda: ops.gemm_nt(dY.transpose(-1, -2), dH.transpose(-1, -2), out=acc, accumulate=True,
                                                     reduce_z1=True, round_out=False)),
            ("dY^T G     ct  ", lambda: ops.gemm_nt(ops._transposed(dY, B * M, U1, Fd).unflatten(0, (B, M)), dHt, out=acc,
                                                     accumulate=True, reduce_z1=True, round_out=False)),
            ("producer   -   ", lambda: ops.gemm_nt(dY, W, out=dH)),
            ("producer   +ct ", lambda: ops.gemm_nt(dY, W, out=dH, ct=ct)),
            ("sx_transpose   ", lambda: ops._transposed(P, B * M, U1, U2))]:
        med, lo, hi = timed(fn, args.rounds, args.reps)
        rows.append((name, med, lo, hi))
    print(torch.cuda.get_device_name(), "(P^T dH and dY^T G: %d-GFLOP products; the transposes of P move 180 MB each way)"
          % round(gf))
    for name, med, lo, hi in rows:
        print("%s %8.3f ms [%.3f, %.3f]" % (name, med, lo, hi))


if __name__ == "__main__":
    main()
