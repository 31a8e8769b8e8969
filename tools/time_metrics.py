"""Time the GPU evaluation metrics (segtran_b200.metrics.calculate_metric_percase) on a generated BraTS-sized case
(240x240x155, 4 classes, float maps on the GPU as test_all_cases holds them) with hd95=False (the reference's columns)
and hd95=True, and the host restatement (scipy, as medpy runs it) on the same case.

    python tools/time_metrics.py [--reps 20] [--host-reps 1] [--seed 101]

GPU: CUDA events around each call after a warm-up, median and range over --reps calls (each call ends with its one
device-to-host copy).  Host: wall time of the restatement with hd95 off and on, with torch's thread count and the core
count.  Prints the device name and power limit read in the same run."""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import metric_oracle as MO  # noqa: E402
from segtran_b200 import metrics as SM  # noqa: E402


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                      # the measurement still names the device below
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | %s" % (torch.cuda.get_device_name(0), q)


def time_gpu(pred, gt, hd95, reps):
    for _ in range(3):
        SM.calculate_metric_percase(pred, gt, 4, hd95=hd95)
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        out = SM.calculate_metric_percase(pred, gt, 4, hd95=hd95)
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return ts, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=1)
    ap.add_argument("--seed", type=int, default=101)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_metrics: needs a GPU")
    print("device:", device_line())
    p, g = MO.brats_like_case(a.seed)
    pc, gc = p.float().cuda(), g.float().cuda()
    for hd95 in (False, True):
        ts, (metric, _) = time_gpu(pc, gc, hd95, a.reps)
        print("gpu  hd95=%-5s  median %.3f ms  min %.3f  max %.3f  (%d calls)  metric %s"
              % (hd95, statistics.median(ts), min(ts), max(ts), a.reps, metric.round(6).tolist()))
    try:
        import scipy  # noqa: F401
    except ImportError:
        print("host: scipy not installed, host restatement not timed")
        return
    for hd95 in (False, True):
        ts = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            metric, _ = MO.calculate_metric_percase(p, g, 4, hd95_on=hd95)
            ts.append(time.perf_counter() - t0)
        print("host hd95=%-5s  median %.3f s  (%d runs; torch threads %d, %d cores; scipy is single-threaded)  metric %s"
              % (hd95, statistics.median(ts), a.host_reps, torch.get_num_threads(), os.cpu_count(),
                 metric.round(6).tolist()))


if __name__ == "__main__":
    main()
