"""Generate tests/golden/tta_*.pt: mirror test-time augmentation from the REAL reference sliding-window functions.

TEST INFRASTRUCTURE ONLY (build container: reads the reference).  Run:  python -m oracle.gen_tta_golden
For every variant m of ``mirror_axes`` (bit i mirrors mirror_axes[i]) the reference's test_util3d.test_single_case or
test_util2d.test_single_batch runs with the seeded, non-mirror-symmetric AsymNet of oracle/tta_oracle.py wrapped as
x -> flip_m(net(flip_m(x))).  The fixture's soft output is the mean of the variants' soft outputs, and its hard masks
come from that mean: the reference's make_brats_pred_consistent and threshold (test_util3d.py:165-170), its arg-max,
or its harden_segmap2d.  To get each variant's average before the BraTS rule, the 3-D calls run with the reference's
make_brats_pred_consistent replaced by the identity.  The reference's 3-D padding branch hands F.pad its pads one
dimension off (test_util3d.py:119-120: the C axis gets the H pads); for the padded volume the generator passes F.pad
the pads in the order the surrounding code intends (H, W, D), as oracle/infer_oracle.py does.  Its accumulators are
allocated with ``device='cuda'``; they are redirected to the CPU.
"""
from __future__ import annotations

import os
import sys

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import gen_eval2d_golden as G2               # noqa: E402
from oracle.tta_oracle import AsymNet, mirror_dims       # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# name: (task, K, image shape [C,H,W,D], orig_patch, input_patch, batch_size, stride_xy, stride_z, mirror_axes)
CASES3D = {
    "tta_3d_brats_pad": ("brats", 4, (4, 18, 40, 14), (24, 24, 16), (16, 16, 12), 3, 6, 6, (0, 1, 2)),
    "tta_3d_brats_2ax": ("brats", 4, (4, 26, 26, 20), (20, 20, 16), (16, 12, 12), 3, 8, 4, (2, 0)),
    "tta_3d_2class": ("other", 2, (2, 22, 22, 16), (12, 12, 10), (12, 12, 10), 4, 6, 6, (1,)),
}
# name: (K, image shape [B,C,H,W], orig_input_size, patch_size, stride, mirror_axes)
CASES2D = {
    "tta_2d_pad_resized": (3, (2, 3, 40, 58), (48, 32), (24, 16), (24, 20), (0, 1)),
    "tta_2d_same_size": (2, (2, 3, 50, 44), (24, 24), (24, 24), (12, 16), (1, 0)),
}


class Mirrored(torch.nn.Module):
    def __init__(self, net, dims):
        super().__init__()
        self.net, self.dims = net, dims

    def forward(self, x):
        if not self.dims:
            return self.net(x)
        return torch.flip(self.net(torch.flip(x, self.dims)), self.dims)


def _cuda_to_cpu(fn):
    def wrapped(*a, **kw):
        if kw.get("device") == "cuda":
            kw["device"] = "cpu"
        return fn(*a, **kw)
    return wrapped


def _pad_hwd(pad_fn):
    def wrapped(x, pad, *a, **kw):
        if x.dim() == 4 and len(pad) == 8 and tuple(pad[:2]) == (0, 0):      # test_util3d.py:119-120
            pad = tuple(pad[2:]) + (0, 0)
        return pad_fn(x, pad, *a, **kw)
    return wrapped


def gen_3d(T3):
    zeros, pad, consistent = torch.zeros, F.pad, T3.make_brats_pred_consistent
    for name, (task, K, shp, orig, inp, bs, sxy, sz, axes) in CASES3D.items():
        torch.manual_seed(len(name) + 70)
        image = torch.randn(*shp) * 2.0
        p = AsymNet.params(K, shp[0], seed=len(name) + 80)
        net = AsymNet(**p)
        softs = []
        torch.zeros, F.pad, T3.make_brats_pred_consistent = _cuda_to_cpu(zeros), _pad_hwd(pad), lambda s, **kw: s
        try:
            for dims in mirror_dims(axes, 2):
                _, soft = T3.test_single_case(Mirrored(net, dims), image, orig, inp, bs, sxy, sz, task, "segtran", K)
                softs.append(soft)
        finally:
            torch.zeros, F.pad, T3.make_brats_pred_consistent = zeros, pad, consistent
        soft = torch.stack(softs).mean(0)
        if task == "brats":
            soft = consistent(soft, is_conservative=False)
            hard = torch.zeros_like(soft)
            hard[1:] = (soft[1:] >= 0.5)
            hard[0] = (hard[1:].sum(dim=0) == 0)
        else:
            hard = torch.argmax(soft, dim=0)
        fx = dict(kind="tta3d", task=task, K=K, image=image, orig_patch=orig, input_patch=inp, batch_size=bs,
                  stride_xy=sxy, stride_z=sz, mirror_axes=axes, net=p, hard=hard, soft=soft)
        torch.save(fx, os.path.join(OUT, name + ".pt"))
        print(name, tuple(hard.shape), float(soft.mean()))


def gen_2d(T2):
    zeros = torch.zeros
    for name, (K, shp, orig, patch, stride, axes) in CASES2D.items():
        torch.manual_seed(len(name) + 90)
        image = torch.randn(*shp) * 2.0
        p = AsymNet.params(K, shp[1], seed=len(name) + 100)
        net = AsymNet(**p)
        softs = []
        torch.zeros = _cuda_to_cpu(zeros)
        try:
            for dims in mirror_dims(axes, 2):
                _, soft = T2.test_single_batch(Mirrored(net, dims), image, orig, patch, stride, "fundus", K, "segtran")
                softs.append(soft)
        finally:
            torch.zeros = zeros
        soft = torch.stack(softs).mean(0)
        hard = T2.harden_segmap2d(soft)
        fx = dict(kind="tta2d", K=K, image=image, orig=orig, patch=patch, stride=stride, mirror_axes=axes, net=p,
                  hard=hard, soft=soft.contiguous())
        torch.save(fx, os.path.join(OUT, name + ".pt"))
        print(name, tuple(hard.shape), hard.dtype, float(soft.mean()))


def main():
    torch.set_num_threads(4)
    T2 = G2._ref_util2d()                      # stubs every module test_util3d needs too
    sys.modules["medpy"].metric = sys.modules["medpy.metric"]
    import test_util3d as T3                   # code/test_util3d.py
    gen_3d(T3)
    gen_2d(T2)


if __name__ == "__main__":
    main()
