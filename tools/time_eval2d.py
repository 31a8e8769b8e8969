"""Time the 2-D evaluation drop-ins against the reference's formulation (oracle/eval2d_oracle.py) on the same GPU:
segtran_b200.inference.test_single_batch at the fundus default (B=6, K=3, 576x576 images, orig_input_size 576,
patch_size 288, stride 288) with an element-wise stand-in net, so only the post-process differs between the two; and
segtran_b200.metrics.calc_batch_metric with vCDR against 576x576 ground truths, from 576x576 soft maps (what
test_single_batch returns) and from 288x288 ones (a resize per image).

    python tools/time_eval2d.py [--reps 20] [--warmup 5] [--seed 7] [--kernels]

CUDA events around each call after --warmup calls, median and range over --reps calls.  Every call of the metric ends
with its device-to-host copy, so its time is the caller's.  test_single_batch has no sync: its "call" time includes the
host's launch gaps, and its "device" time is taken with a sleep kernel queued ahead of the start event, so that every
launch of the call is already queued when the GPU reaches it.  --kernels adds, in a separate profiled pass, each
library kernel's time and the bandwidth its minimum traffic implies.  Prints the device name and power limit read in the
same run."""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import eval2d_oracle as E  # noqa: E402
from segtran_b200 import inference as SI  # noqa: E402
from segtran_b200 import metrics as SM  # noqa: E402
from tests.helpers import AffinePickNet  # noqa: E402


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                      # the measurement still names the device below
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | %s" % (torch.cuda.get_device_name(0), q)


def time_calls(fn, reps, warmup, queue_ahead=False):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if queue_ahead:
            torch.cuda._sleep(4_000_000)                        # ~2 ms of GPU time while the host queues the call
        s.record()
        out = fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return ts, out


def report(name, ts):
    print("%-44s median %8.3f ms  min %8.3f  max %8.3f  (%d calls)" % (name, statistics.median(ts), min(ts), max(ts),
                                                                    len(ts)))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_eval2d: needs a GPU")
    print("device:", device_line())
    torch.manual_seed(a.seed)
    B, K, S = 6, 3, 576
    image = (torch.randn(B, 3, S, S) * 2).cuda()
    net = AffinePickNet([1.2, 1.6, 2.0], [-0.4, -0.1, 0.2], [0, 1, 2]).cuda()
    args = ((S, S), (288, 288), (288, 288), "fundus", K, "segtran")

    ours = lambda: SI.test_single_batch(net, image, *args)              # noqa: E731
    ref = lambda: E.test_single_batch(net, image, *args)                # noqa: E731
    for mode, ahead in (("call", False), ("device", True)):
        ts, (hard, soft) = time_calls(ours, a.reps, a.warmup, ahead)
        t_new = report("test_single_batch %-6s segtran_b200" % mode, ts)
        ts, (ref_hard, ref_soft) = time_calls(ref, a.reps, a.warmup, ahead)
        t_ref = report("test_single_batch %-6s reference formulation" % mode, ts)
        print("  speed-up %.2fx; max |soft - ref| %.2e; hard maps differ at %d of %d elements"
              % (t_ref / t_new, float((soft - ref_soft).abs().max()), int((hard != ref_hard).sum()), hard.numel()))

    gt = E.fundus_like_gt(B, S, S, seed=a.seed).cuda()
    for h in (S, S // 2):
        pred = E.soft_from_gt(E.fundus_like_gt(B, S, S, a.seed, jitter=0.3, jitter_seed=a.seed + 1), h, h,
                              seed=a.seed + 2).cuda()
        ts, out = time_calls(lambda: SM.calc_batch_metric(pred, gt, K, do_calc_vcdr_error=True), a.reps, a.warmup)
        t_new = report("calc_batch_metric vCDR %dx%d->%d  segtran_b200" % (h, h, S), ts)
        ts, ref = time_calls(lambda: E.calc_batch_metric(pred, gt, K, do_calc_vcdr_error=True), a.reps, a.warmup)
        t_ref = report("calc_batch_metric vCDR %dx%d->%d  reference" % (h, h, S), ts)
        print("  speed-up %.2fx; max |metric - ref| %.2e" % (t_ref / t_new, float(np.abs(out - ref).max())))
    if a.kernels:
        kernel_rates(ours, lambda: SM.calc_batch_metric(pred, gt, K, do_calc_vcdr_error=True), B, K, S, pred.shape[-1])


def kernel_rates(sw, metric, B, K, S, h):
    """mean time per launch of each sx_eval2d kernel (torch.profiler, 10 calls) and the minimum HBM traffic over it"""
    from torch.profiler import ProfilerActivity, profile
    f = 4
    traffic = {"sw2d_accumulate": B * K * (2 * S * S + (S // 2) ** 2) * f + 2 * S * S * f,   # preds RMW, scores, cnt RMW
               "sw2d_finalize": B * K * S * S * 3 * f + S * S * f,                             # preds, soft, hard; cnt
               "eval2d_counts": B * (K - 1) * (S * S + h * h) * f}                             # gt and pred classes >= 1
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            sw()
            metric()
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        for name, nbytes in traffic.items():
            if name in ev.key and ev.count:
                us = ev.self_device_time_total / ev.count
                print("kernel %-16s %8.2f us per launch  %6.1f MB  %6.2f TB/s" % (name, us, nbytes / 1e6, nbytes / us / 1e6))


if __name__ == "__main__":
    main()
