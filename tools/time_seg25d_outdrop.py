"""Time the 2.5-D --outdrop head's forward + backward at the full 2.5-D shape against the eager formulation on the same GPU.

Shape: input [1,4,112,112,96] with eff-b3 widths: out-FPN map [96, 136, 56, 56] (slice-major), fused tokens [1, 9408, 1536]
on the (14, 14, 48) grid, 2 classes, D_pool_K = 2, dropout p = 0.2, logits [1, 2, 112, 112, 96].  Cases: --upd conv
(interleaved depth unfold) and --upd interpolate (linear x 2 along depth).
  segtran_b200  ops.seg_head_slices_dropout: slice-major addend, bridge GEMM, (upsampleD GEMM), dropout-head kernels
  eager         the reference's formulation (segtran25d.py:351-377, :464-477) in stock PyTorch: permute to
                [B,C,H1,W1,D2], Conv3d bridge + trilinear tokens, Conv3d upsampleD + view/permute/reshape or trilinear,
                nn.Dropout, out_conv3d, trilinear to the input size
Each figure is the median over --rounds rounds of --iters forward + backward calls timed with CUDA events after warm-up;
the peak is torch.cuda.max_memory_allocated above the inputs during one call.

    python tools/time_seg25d_outdrop.py [--rounds 5] [--iters 5]

Prints the device name and its power limit, read in the same run, next to the numbers."""
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

B, D2, CF, FD, K, DK, H1 = 1, 96, 136, 1536, 2, 2, 56
GRID = (14, 14, 48)
OUT = (112, 112, 96)
P = 0.2


def make(upd):
    g = torch.Generator(device="cuda").manual_seed(0)
    r = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).requires_grad_()   # noqa: E731
    Fo = FD // DK if upd == "conv" else FD
    t = dict(curr=r(B * D2, CF, H1, H1), vf=r(B, GRID[0] * GRID[1] * GRID[2], FD), Wb=r(FD, CF, 1, 1, 1, sc=0.05),
             bb=r(FD, sc=0.1), Wc=r(K, Fo, 1, 1, 1, sc=0.03), bc=r(K, sc=0.1), Wu=None, bu=None)
    if upd == "conv":
        t["Wu"], t["bu"] = r(Fo * DK, FD, 1, 1, 1, sc=0.03), r(Fo * DK, sc=0.1)
    return t


def ours(t, upd):
    return ops.seg_head_slices_dropout(t["curr"], t["vf"], GRID, t["Wb"], t["bb"], t["Wc"], t["bc"], OUT, P, DK, upd,
                                       Wu=t["Wu"], bu=t["bu"])


def eager(t, upd):
    H2, W2, D3 = GRID
    vol = t["curr"].view(B, D2, CF, H1, H1).permute(0, 2, 3, 4, 1)
    vmap = t["vf"].view(B, H2, W2, D3, FD).permute(0, 4, 1, 2, 3)
    x = F.conv3d(vol, t["Wb"], t["bb"]) + F.interpolate(vmap, size=(H1, H1, D2), mode="trilinear", align_corners=False)
    if upd == "conv":
        y = F.conv3d(x, t["Wu"], t["bu"])
        y = y.view((B, FD // DK, DK) + tuple(x.shape[2:])).permute(0, 1, 3, 4, 5, 2)
        x = y.reshape(tuple(y.shape[:4]) + (-1,))
    else:
        x = F.interpolate(x, size=(H1, H1, D2 * DK), mode="trilinear", align_corners=False)
    x = F.dropout(x, P, training=True)
    s = F.conv3d(x, t["Wc"], t["bc"])
    return F.interpolate(s, size=OUT, mode="trilinear", align_corners=False)


def call(fn, t, upd, G):
    fn(t, upd).backward(G)


def time_case(fn, t, upd, G, rounds, iters):
    for _ in range(2):
        call(fn, t, upd, G)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    call(fn, t, upd, G)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    times = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            call(fn, t, upd, G)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / iters)
    return statistics.median(times), min(times), max(times), peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_seg25d_outdrop: needs a CUDA device (no CPU timing)")
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:                                    # noqa: BLE001  (no nvidia-smi: report it as unknown)
        pl = "unknown"
    print("device: %s, power limit: %s" % (name, pl))
    print("precision: %s, p = %.2f, curr [%d,%d,%d,%d], tokens %s x %d, logits [%d,%d,%d,%d,%d]"
          % (ops.get_precision(), P, B * D2, CF, H1, H1, GRID, FD, B, K, *OUT))
    for upd in ("conv", "interpolate"):
        t = make(upd)
        G = torch.randn(B, K, *OUT, device="cuda")
        for label, fn in (("segtran_b200", ours), ("eager", eager)):
            for v in t.values():
                if v is not None:
                    v.grad = None
            med, lo, hi, peak = time_case(fn, t, upd, G, args.rounds, args.iters)
            print("--upd %-11s %-12s  fwd+bwd %8.2f ms (%.2f-%.2f)  peak above inputs %6.2f GiB"
                  % (upd, label, med, lo, hi, peak / 2 ** 30))
        del t, G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
