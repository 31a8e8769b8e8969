"""Time Gaussian window blending (``gaussian_sigma_scale`` of segtran_b200.inference) against the plain average, with and
without mirror test-time augmentation, on the same GPU.

    python tools/time_gaussian_blend.py [--reps 5] [--warmup 1]

3-D: test_single_case on a [4,240,240,155] volume (a whole BraTS case) with the 112^3 window and the driver's strides
(half the window, 56 / 56; 4 x 4 x 2 = 32 windows), batch_size 4, BraTS post-process.  2-D: test_single_batch at the
REFUGE size (B=6, K=3, 576x576 images, orig_input_size 576, patch 288, stride 288).  Both use the element-wise stand-in
net of the TTA fixtures, so the times are the sliding window itself rather than a network.  Each arm runs plain and
gaussian_sigma_scale=0.125, with mirror_axes=() and with every axis.  Times are CUDA events around a call after
--warmup calls, median over --reps.  Then the accumulate kernel alone: CUDA events around 200 back-to-back
sx_sw_accumulate (one 112^3 window, K=4) or sx_sw2d_accumulate (288^2 scores upsampled to 576^2, B=6, K=3) launches,
unweighted and weighted.  Prints the device name and power limit read in the same run."""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.tta_oracle import AsymNet  # noqa: E402
from segtran_b200 import _lib as L  # noqa: E402
from segtran_b200 import inference as SI  # noqa: E402

S = 0.125


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | %s" % (torch.cuda.get_device_name(0), q)


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return statistics.median(ts), min(ts), max(ts)


def arms(name, run, axes, reps, warmup):
    print("\n%s" % name)
    for ax in ((), axes):
        plain = timed(lambda: run(ax, None), reps, warmup)
        gauss = timed(lambda: run(ax, S), reps, warmup)
        for k, (med, lo, hi) in (("plain", plain), ("gaussian %.3f" % S, gauss)):
            print("  mirror_axes=%-10s %-15s median %9.2f ms  (%8.2f - %8.2f)" % (ax, k, med, lo, hi))
        print("  mirror_axes=%-10s gaussian - plain %+8.2f ms (%+.1f%%)" % (ax, gauss[0] - plain[0],
                                                                          100 * (gauss[0] / plain[0] - 1)))


def kernel_loop(name, call, wts, n=200, reps=5):
    st = torch.cuda.current_stream().cuda_stream

    def loop(weighted):
        for _ in range(n):
            L.call(*call(wts if weighted else None, st))

    res = {}
    for weighted in (False, True, False, True):                 # alternate the two, keep the last of each
        loop(weighted)
        ts = []
        for _ in range(reps):
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            loop(weighted)
            e.record()
            torch.cuda.synchronize()
            ts.append(s.elapsed_time(e) * 1000 / n)
        res[weighted] = statistics.median(ts)
    print("  %-48s unweighted %8.1f us   weighted %8.1f us per launch" % (name, res[False], res[True]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_gaussian_blend.py measures on the GPU"
    print(device_line())

    image3 = torch.randn(4, 240, 240, 155, device="cuda")
    net3 = AsymNet(**AsymNet.params(4, 4, seed=7))

    def run3(axes, s):
        return SI.test_single_case(net3, image3, (112, 112, 112), (112, 112, 112), 4, 56, 56, "brats", "segtran", 4,
                                   mirror_axes=axes, gaussian_sigma_scale=s)

    arms("3-D BraTS [4,240,240,155], window 112^3, stride 56/56, batch_size 4", run3, (0, 1, 2), a.reps, a.warmup)

    image2 = torch.randn(6, 3, 576, 576, device="cuda")
    net2 = AsymNet(**AsymNet.params(3, 3, seed=7))

    def run2(axes, s):
        return SI.test_single_batch(net2, image2, (576, 576), (288, 288), (288, 288), "fundus", 3, "segtran",
                                    mirror_axes=axes, gaussian_sigma_scale=s)

    arms("2-D REFUGE [6,3,576,576], orig 576, patch 288, stride 288", run2, (0, 1), a.reps, a.warmup)

    print("\naccumulate kernels alone")
    d = (112, 112, 112)
    sc3 = torch.randn((4,) + d, device="cuda")
    pr3 = torch.zeros((4, 240, 240, 155), device="cuda")
    cn3 = torch.zeros((240, 240, 155), device="cuda")
    tab3, wts3 = SI._window_weights(d, S, "cuda")
    kernel_loop("sx_sw_accumulate 112^3 window, K=4",
                lambda wts, st: ("sx_sw_accumulate", sc3.data_ptr(), 4, *d, pr3.data_ptr(), cn3.data_ptr(), 240, 240,
                                 155, 56, 56, 43, 0, wts, st), wts3)
    sc2 = torch.randn(6, 3, 288, 288, device="cuda")
    pr2 = torch.zeros(6, 3, 576, 576, device="cuda")
    cn2 = torch.zeros(576, 576, device="cuda")
    tab2, wts2 = SI._window_weights((576, 576), S, "cuda")
    kernel_loop("sx_sw2d_accumulate 288^2 -> 576^2, B=6, K=3",
                lambda wts, st: ("sx_sw2d_accumulate", sc2.data_ptr(), 6, 3, 288, 288, 576, 576, pr2.data_ptr(),
                                 cn2.data_ptr(), 576, 576, 0, 0, 0, wts, st), wts2)
    del tab3, tab2


if __name__ == "__main__":
    main()
