"""Time the TF32 products that read a K-major copy of a small operand (ops.set_kmajor_copies) against the same product on
the MN-major view, at cfg-4 shapes (Segtran3d BraTS 112^3, batch 4: 2744 tokens, 1024 attractors, 4 modes of 1024
channels, key width 256 per mode):
  pv          squeeze-out G = gelu(P V' + bm) with dropout, P [4,4,2744,1024], V' [4,1024,4*1024]
  dH          squeeze-out dH = mask * (dY Wo) * gelu'(H) with the bias-gradient column sums, Wo [4,1024,1024]
  dQ          squeeze-out dQ = dS K / sqrt(d), dS [4,4,2744,1024], K [4,1024,4*256]
  dx_tok      token-row Linear dX = dY W, dY [10976,1024], W [1024,1024]
  dx_attr     attractor-row Linear dX = dY W, dY [4096,1024], W [1024,1024]
  dx_ffn      attractor-row Linear dX = dY W, dY [4096,4096], W [4096,1024]
"new" includes building the copy (sx_transpose).  Each round times --iters calls of the old and then of the new form
with CUDA events; rounds alternate which goes first, and the median over --rounds rounds is printed.

    python tools/time_kmajor_operands.py [--rounds 7] [--iters 20]

Prints the device name and its power limit next to the numbers (they are part of the measurement)."""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from segtran_b200 import ops  # noqa: E402

B, U1, U2, M, FD, D = 4, 2744, 1024, 4, 1024, 256


def tf32(*shape, scale=1.0):
    return ops.round_tf32(torch.randn(*shape, device="cuda") * scale)


def cases():
    P = tf32(B, M, U1, U2, scale=0.03)
    vp = tf32(B, U2, M * FD)
    bm = torch.randn(FD, device="cuda")
    G = torch.empty(B, M, U1, FD, device="cuda")
    H = torch.empty_like(G)
    dY = tf32(B, M, U1, FD)
    Wr = tf32(M, FD, FD, scale=0.03)
    dH = torch.empty_like(G)
    dbm = torch.zeros(FD, device="cuda")
    k = tf32(B, U2, M * D)
    dq = torch.empty(B, U1, M * D, device="cuda")
    lin = {name: (tf32(R, O), tf32(O, I, scale=0.03)) for name, R, O, I in
           (("dx_tok", B * U1, 1024, 1024), ("dx_attr", B * U2, 1024, 1024), ("dx_ffn", B * U2, 4096, 1024))}

    def pv():
        ops.gemm_nt(P, ops._head_cols(vp, B, U2, M, FD, ops._kmajor_copies()), out=G, bias=bm, gelu=True, preact=H, drop_p=0.2, seed=7)

    def dh():
        ops.gemm_nt(dY, ops._weight_t(Wr, M, FD, FD).unsqueeze(0), out=dH, gelu_bwd=H, drop_p=0.2, seed=7)
        ops.colsum(dH.view(-1, FD), out=dbm)

    def dqf():
        ops.gemm_nt(P, ops._head_cols(k, B, U2, M, D, ops._kmajor_copies()), out=dq.view(B, U1, M, D).permute(0, 2, 1, 3),
                    alpha=0.0625, round_out=False, split_k=1)

    out = {"pv": pv, "dH": dh, "dQ": dqf}
    for name, (dy, W) in lin.items():
        out[name] = (lambda dy=dy, W=W: ops.gemm_nt(dy, ops._weight_t(W, 1, *W.shape)[0], round_out=False))
    return out


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    ops.set_precision("tf32")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print("device: %s (power limit %s)" % tuple((smi[0].split(", ") + ["?", "?"])[:2]) if smi else "device: ?")
    fns = cases()

    def with_copies(on, fn):
        def run():
            ops.set_kmajor_copies(on)
            fn()
        return run

    print("%-8s %10s %10s %8s" % ("site", "old ms", "new ms", "saved"))
    total = 0.0
    for name, fn in fns.items():
        old, new = with_copies(False, fn), with_copies(True, fn)
        for f in (old, new):
            timed(f, 3)
        to, tn = [], []
        for r in range(args.rounds):
            for f, acc in ((old, to), (new, tn)) if r % 2 == 0 else ((new, tn), (old, to)):
                acc.append(timed(f, args.iters))
        mo, mn = statistics.median(to), statistics.median(tn)
        total += mo - mn
        print("%-8s %10.3f %10.3f %8.3f" % (name, mo, mn, mo - mn))
    ops.set_kmajor_copies(True)
    print("sum of per-launch savings: %.3f ms (multiply by each site's launches per step)" % total)


if __name__ == "__main__":
    main()
