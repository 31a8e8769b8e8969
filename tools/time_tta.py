"""Time mirror test-time augmentation (``mirror_axes`` of segtran_b200.inference) against the user-side formulation,
the net wrapped as x -> flip_m(net(flip_m(x))) with torch.flip and one plain call per variant, on the same GPU.

    python tools/time_tta.py [--reps 3] [--warmup 1]

3-D: test_single_case on a [4,160,192,144] volume (a BraTS case cropped to the brain) with the BraTS window
(orig = input patch 112x112x96, stride 56 / 40, batch_size 4, 18 windows), Segtran3d at the bench's cfg-4 widths with
seeded random weights.  Its backbone is a stand-in (average pooling to the I3D endpoints' strides plus a seeded 1x1x1
convolution to their widths), because the I3D weights are not part of the project.  2-D: test_single_batch at the REFUGE
size (B=6, K=3, 576x576 images, orig_input_size 576, patch 288) with an element-wise stand-in net, so its times are the
sliding window and the augmentation alone.  Each arm: plain (mirror_axes=()), TTA over every axis, and the wrapped
formulation; "net" is the 2^k forward calls of the net alone on batches of the same shapes, so "beyond the net calls" =
arm - net.  Times are CUDA events around a call after --warmup calls, median over --reps; peak memory is
torch.cuda.max_memory_allocated above what was allocated before the call.  Prints the device name and power limit read
in the same run."""
from __future__ import annotations

import argparse
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from oracle.tta_oracle import AsymNet  # noqa: E402
from segtran_b200 import inference as SI  # noqa: E402


def device_line():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | %s" % (torch.cuda.get_device_name(0), q)


class PooledFeat3d(torch.nn.Module):
    """Stand-in I3D: endpoint i = seeded 1x1x1 conv of the frames-first input average-pooled by STRIDES[i] (D, H, W)."""
    STRIDES = [(2, 2, 2), (2, 2, 2), (2, 4, 4), (4, 8, 8), (8, 16, 16)]
    KEYS = ["MaxPool3d_2a_3x3", "Conv3d_2c_3x3", "Mixed_3c", "Mixed_4f", "Mixed_5c"]

    def __init__(self, dims):
        super().__init__()
        self.convs = torch.nn.ModuleList(torch.nn.Conv3d(3, d, 1) for d in dims)

    def extract_features(self, x):
        return {k: conv(F.avg_pool3d(x, s)) for k, s, conv in zip(self.KEYS, self.STRIDES, self.convs)}


def segtran3d_cfg4():
    import segtran_b200.networks.segtran3d as M
    import segtran_b200.networks.segtran_shared as S
    c = bench.CONFIGS[4]
    torch.manual_seed(1337)
    cfg = M.Segtran3dConfig()
    cfg.update_config(bench.model_args(c, "cuda", 0.0))
    net = M.Segtran3d(cfg, backbone=PooledFeat3d(S.bb2feat_dims["i3d"]))
    net.scales_printed = True
    return net.cuda().eval()


class Mirrored(torch.nn.Module):
    def __init__(self, net, dims):
        super().__init__()
        self.net, self.dims = net, dims

    def forward(self, x):
        return torch.flip(self.net(torch.flip(x, self.dims)), self.dims) if self.dims else self.net(x)


class Recorder(torch.nn.Module):
    def __init__(self, net):
        super().__init__()
        self.net, self.shapes = net, []

    def forward(self, x):
        self.shapes.append(tuple(x.shape))
        return self.net(x)


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts, peaks = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
        peaks.append(torch.cuda.max_memory_allocated() - base)
        del out
    return statistics.median(ts), min(ts), max(ts), max(peaks)


def arms(name, run, net, dims_of_variants, reps, warmup):
    """run(net, mirror_axes) -> outputs; prints plain, TTA, wrapped and net-only times."""
    rec = Recorder(net)
    run(rec, ())
    shapes = rec.shapes
    batches = [torch.randn(s, device="cuda") for s in shapes]
    nv = len(dims_of_variants)

    def net_only():
        with torch.no_grad():
            for _ in range(nv):
                for b in batches:
                    net(b)

    def wrapped():
        acc = None
        for dims in dims_of_variants:
            _, soft = run(Mirrored(net, dims), ())
            acc = soft if acc is None else acc.add_(soft)
        return acc.div_(nv)

    axes = tuple(range(len(shapes[0]) - 2))
    res = {"plain": timed(lambda: run(net, ()), reps, warmup),
           "TTA %s" % (axes,): timed(lambda: run(net, axes), reps, warmup),
           "wrapped with torch.flip": timed(wrapped, reps, warmup),
           "net alone, %d variants" % nv: timed(net_only, reps, warmup)}
    print("\n%s: %d net calls per variant, batch shapes %s" % (name, len(shapes), sorted(set(shapes))))
    net_ms = res["net alone, %d variants" % nv][0]
    for k, (med, lo, hi, pk) in res.items():
        extra = "" if k.startswith("net") or k == "plain" else "   beyond the net calls %8.2f ms" % (med - net_ms)
        print("  %-26s median %9.2f ms  (%8.2f - %8.2f)  peak %7.0f MB%s" % (k, med, lo, hi, pk / 2**20, extra))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_tta.py measures on the GPU"
    print(device_line())
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True

    net3 = segtran3d_cfg4()
    image3 = torch.randn(4, 160, 192, 144, device="cuda")

    def run3(net, axes):
        return SI.test_single_case(net, image3, (112, 112, 96), (112, 112, 96), 4, 56, 40, "brats", "segtran", 4,
                                   mirror_axes=axes)

    variants3 = [[2 + a for a in range(3) if m >> a & 1] for m in range(8)]
    arms("3-D Segtran3d cfg-4 widths, [4,160,192,144], batch_size 4", run3, net3, variants3, a.reps, a.warmup)

    net2 = AsymNet(**AsymNet.params(3, 3, seed=7))
    image2 = torch.randn(6, 3, 576, 576, device="cuda")

    def run2(net, axes):
        return SI.test_single_batch(net, image2, (576, 576), (288, 288), (288, 288), "fundus", 3, "segtran",
                                    mirror_axes=axes)

    variants2 = [[2 + a for a in range(2) if m >> a & 1] for m in range(4)]
    arms("2-D REFUGE [6,3,576,576], patch 288, element-wise stand-in net", run2, net2, variants2, a.reps, a.warmup)


if __name__ == "__main__":
    main()
