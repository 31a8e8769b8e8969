"""Time the class head without the out-FPN (out_fpn_layers == in_fpn_layers), ops.direct_head, against stock PyTorch
(F.conv_transpose2d/3d + F.interpolate, as the reference runs it) on the same GPU, forward and forward + backward:
  cfg 4  B = 4, tokens on a 14^3 grid, C = 1024, K = 4, logits [4,4,112,112,112]  (ConvTranspose3d (2,2,1) + trilinear)
  cfg 1  B = 2, tokens on a 36^2 grid, C = 1792, K = 3, logits [2,3,288,288]      (ConvTranspose2d 2 + bilinear)
Reports the median time per call over --rounds rounds of --iters calls (CUDA events), the agreement of the two logits,
and the achieved bytes/s against a lower bound on the HBM traffic computed from the shapes: the forward reads the
tokens X and writes the logits; the backward reads the logit gradient and X and writes dX (the weights, the sub-pixel
scores and their gradient are small and not counted).

    python tools/time_direct_head.py [--rounds 5] [--iters 10]

Prints the device name and its power limit next to the numbers (they are part of the measurement)."""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from segtran_b200 import ops  # noqa: E402

CFGS = {"cfg4": dict(B=4, grid=(14, 14, 14), C=1024, K=4, out=(112, 112, 112)),
        "cfg1": dict(B=2, grid=(36, 36), C=1792, K=3, out=(288, 288))}


def make(c):
    g = torch.Generator(device="cuda").manual_seed(0)
    N = 1
    for v in c["grid"]:
        N *= v
    X = torch.randn(c["B"], N, c["C"], device="cuda", generator=g).requires_grad_()
    Wt = (torch.randn(c["C"], c["K"], 2, 2, *((1,) if len(c["grid"]) == 3 else ()), device="cuda", generator=g)
          * 0.03).requires_grad_()
    bt = torch.randn(c["K"], device="cuda", generator=g).requires_grad_()
    G = torch.randn((c["B"], c["K"]) + c["out"], device="cuda", generator=g)
    return X, Wt, bt, G


def ours(c, X, Wt, bt):
    return ops.direct_head(X, c["grid"], Wt, bt, c["out"])


def stock(c, X, Wt, bt):
    B, N, C = X.shape
    m = X.transpose(1, 2).reshape(B, C, *c["grid"])
    if len(c["grid"]) == 3:                                  # tokens (D2,H2,W2) -> (H2,W2,D2), as the reference permutes
        s = F.conv_transpose3d(m.permute(0, 1, 3, 4, 2), Wt, bt, stride=(2, 2, 1))
        return F.interpolate(s, size=c["out"], mode="trilinear", align_corners=False)
    s = F.conv_transpose2d(m, Wt, bt, stride=2)
    return F.interpolate(s, size=c["out"], mode="bilinear", align_corners=False)


def timed(fn, rounds, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / iters)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_direct_head.py needs a GPU")
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:                                    # noqa: BLE001  (no nvidia-smi: report it as unknown)
        pl = "unknown"
    print("device: %s, power limit: %s" % (torch.cuda.get_device_name(0), pl))
    torch.backends.cudnn.allow_tf32 = False             # the stock arm in fp32, like the head
    for name, c in CFGS.items():
        X, Wt, bt, G = make(c)
        with torch.no_grad():
            yo, ys = ours(c, X, Wt, bt), stock(c, X, Wt, bt)
            agree = float((yo - ys).abs().max() / ys.abs().max())
        x_bytes, y_bytes = 4.0 * X.numel(), 4.0 * G.numel()
        fwd_bytes, bwd_bytes = x_bytes + y_bytes, y_bytes + 2 * x_bytes
        print("[%s] X %s (%.1f MB), logits %s (%.1f MB); logits max|ours - stock| / max|stock| = %.2e"
              % (name, tuple(X.shape), x_bytes / 1e6, tuple(G.shape), y_bytes / 1e6, agree))
        for arm, fn in (("direct_head", ours), ("stock", stock)):
            def fwd():
                with torch.no_grad():
                    fn(c, X, Wt, bt)

            def fwd_bwd():
                torch.autograd.grad(fn(c, X, Wt, bt), (X, Wt, bt), G)

            tf, tb = timed(fwd, a.rounds, a.iters), timed(fwd_bwd, a.rounds, a.iters)
            print("   %-11s fwd %8.3f ms (%6.0f GB/s of %.0f MB)   fwd+bwd %8.3f ms (%6.0f GB/s of %.0f MB)"
                  % (arm, tf, fwd_bytes / tf / 1e6, fwd_bytes / 1e6, tb, (fwd_bytes + bwd_bytes) / tb / 1e6,
                     (fwd_bytes + bwd_bytes) / 1e6))


if __name__ == "__main__":
    main()
