"""Time the segmentation head's forward + backward at cfg-4 head shapes (curr [4,832,56,56,56], fused tokens
[4,2744,1024] on a 14^3 grid, 4 classes, D_pool_K = 2, logits [4,4,112,112,112]) for four cases:
  default             collapsed head, depth 'interp'
  --upd conv          out_fpn_upsampleD folded into the collapsed head
  --outdrop p=0.2     dropout head (csrc/sx_head_drop.cu), depth 'interp'
  both                --upd conv and --outdrop: Y2 = Wu Y + bu, then the dropout head with the unfold map
Reports the time per forward + backward (median of --rounds rounds of --iters calls), the peak memory allocated, the
achieved TFLOP/s of the sx_gemm calls and the GB/s of the dropout-head kernels against a byte model from shapes (forward:
read the source map once, write the scores; backward: read the source map and its neighbour slices' taps once, write
its gradient, read the score gradient), each from CUDA events around every C-ABI call in a run of its own.

    python tools/time_head_options.py [--rounds 3] [--iters 5]

Prints the device name and its power limit next to the numbers (they are part of the measurement)."""
from __future__ import annotations

import argparse
import contextlib
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from segtran_b200 import _lib, ops  # noqa: E402

B, CF, FD, K, DK, D1, GRID = 4, 832, 1024, 4, 2, 56, (14, 14, 14)
OUT = (112, 112, 112)


def make():
    g = torch.Generator(device="cuda").manual_seed(0)
    r = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).requires_grad_()   # noqa: E731
    return dict(curr=r(B, CF, D1, D1, D1), vf=r(B, GRID[0] * GRID[1] * GRID[2], FD), Wb=r(FD, CF, 1, 1, 1, sc=0.03),
                bb=r(FD, sc=0.1), Wc=r(K, FD, 1, 1, 1, sc=0.03), bc=r(K), Wc2=r(K, FD // DK, 1, 1, 1, sc=0.03),
                Wu=r(FD, FD, 1, 1, 1, sc=0.03), bu=r(FD, sc=0.1))


def run(case, t, G):
    if case == "default":
        y = ops.seg_head(t["curr"], t["vf"], GRID, t["Wb"], t["bb"], t["Wc"], t["bc"], OUT, d_pool_k=DK)
    elif case == "upd_conv":
        Wf, bf = ops.fold_unfold(t["Wc2"], t["bc"], t["Wu"], t["bu"], DK)
        y = ops.seg_head(t["curr"], t["vf"], GRID, t["Wb"], t["bb"], Wf, bf, OUT, d_unfold=DK)
    elif case == "outdrop":
        y = ops.seg_head_dropout(t["curr"], t["vf"], GRID, t["Wb"], t["bb"], t["Wc"], t["bc"], OUT, 0.2, d_pool_k=DK)
    else:
        y = ops.seg_head_dropout(t["curr"], t["vf"], GRID, t["Wb"], t["bb"], t["Wc2"], t["bc"], OUT, 0.2, d_pool_k=DK,
                                 upsample_d="conv", Wu=t["Wu"], bu=t["bu"])
    y.backward(G)


class Hook:
    """CUDA events around every C-ABI call; sx_gemm flops and dropout-head bytes from the call's arguments."""

    def __init__(self):
        self.rec = []

    @contextlib.contextmanager
    def __call__(self, name, args):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        yield
        e1.record()
        work = 0.0
        a = getattr(args[0], "_obj", None) if args else None
        if name == "sx_gemm" and a is not None:
            work = 2.0 * a.M * a.N * a.K * a.Z0 * a.Z1
        elif name.startswith("sx_head_dropout") and a is not None:
            src = 4.0 * a.B * a.Fs * a.Ds * a.HW
            Do = a.Ds if a.dmap == _lib.SX_HEAD_DMAP_NONE else a.Ds * a.Dk
            ls = 4.0 * a.B * a.K * Do * a.HW
            work = src + ls if name.endswith("fwd") else 2 * src + ls
        self.rec.append((name, e0, e1, work))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:                                    # noqa: BLE001  (no nvidia-smi: report it as unknown)
        pl = "unknown"
    print("device: %s, power limit: %s" % (name, pl))
    t = make()
    G = torch.randn(B, K, *OUT, device="cuda")
    cases = ["default", "upd_conv", "outdrop", "both"]
    times = {c: [] for c in cases}
    peaks = {}
    for c in cases:                                       # warm-up (and peak memory)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run(c, t, G)
        torch.cuda.synchronize()
        peaks[c] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        for v in t.values():
            v.grad = None
    for _ in range(a.rounds):
        for c in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                run(c, t, G)
                for v in t.values():
                    v.grad = None
            e1.record()
            torch.cuda.synchronize()
            times[c].append(e0.elapsed_time(e1) / a.iters)
    base_ms = statistics.median(times["default"])
    for c in cases:
        ms = statistics.median(times[c])
        print("%-9s fwd+bwd %8.2f ms  (x%.2f of default)  peak extra memory %.2f GiB" % (c, ms, ms / base_ms, peaks[c]))
    for c in cases:
        h = Hook()
        _lib.set_hook(h)
        run(c, t, G)
        _lib.set_hook(None)
        torch.cuda.synchronize()
        for v in t.values():
            v.grad = None
        agg = {}
        for n, e0, e1, w in h.rec:
            ms = e0.elapsed_time(e1)
            s = agg.setdefault(n, [0, 0.0, 0.0])
            s[0] += 1
            s[1] += ms
            s[2] += w
        print("[%s] per entry point (ms, calls):" % c)
        for n, (cnt, ms, w) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            extra = ""
            if n == "sx_gemm":
                extra = "  %.1f TFLOP/s (%.2f TFLOP)" % (w / ms / 1e9, w / 1e12)
            elif n.startswith("sx_head_dropout"):
                extra = "  %.0f GB/s of the byte model (%.2f GB)" % (w / ms / 1e6, w / 1e9)
            print("   %-28s %8.3f ms %3d%s" % (n, ms, cnt, extra))


if __name__ == "__main__":
    main()
