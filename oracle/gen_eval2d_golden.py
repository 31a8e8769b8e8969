"""Generate tests/golden/eval2d.pt by running the REAL reference 2-D evaluation (build container only: reads the reference).

TEST INFRASTRUCTURE ONLY.  Run:  python -m oracle.gen_eval2d_golden
test_util2d (code/test_util2d.py) imports on a CPU-only host once imgaug (with augmenters and
augmentables.segmaps.SegmentationMapsOnImage), matplotlib (with cm), and the stubs of gen_golden.gen_infer are in
sys.modules; its ``torch.zeros(..., device='cuda')`` accumulator (:183) is redirected to the CPU.  The net is the
element-wise AffinePickNet of tests/helpers.py, so the fixtures pin the sliding-window logic, not a network.
(a) sw: test_single_batch on a padded K=3 fundus-like batch with upsampled scores and overlapping windows along W, a
    K=2 polyp-like batch with patch_size == orig_input_size and overlapping windows on both axes, and a single ×2
    upsampled window (the shape of the REFUGE default, scaled down).
(b) metric: calc_batch_metric with and without vCDR on elliptical disc-containing-cup ground truths larger than the
    prediction, a prediction already at GT size, a polyp-like K=2 batch, edge cases (a prediction without a cup, a
    ground truth without a disc, an empty class), and a list input of two sizes.  Ground truths are stored as uint8.
"""
from __future__ import annotations

import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import eval2d_oracle as E                   # noqa: E402
from oracle import ref_import as R                      # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# key: (K, image shape, orig_input_size, patch_size, stride)
SW = {"fundus_pad": (3, (2, 3, 40, 58), (48, 32), (24, 16), (24, 20)),
      "polyp_overlap": (2, (2, 3, 50, 44), (24, 24), (24, 24), (12, 16)),
      "single_x2": (3, (2, 3, 48, 48), (48, 48), (24, 24), (48, 48))}


def _ref_util2d():
    R.load()
    stubs = ("h5py", "nibabel", "medpy", "medpy.metric", "common_util", "tqdm", "imgaug", "imgaug.augmenters",
             "imgaug.augmentables", "imgaug.augmentables.segmaps", "matplotlib", "matplotlib.cm")
    for name in stubs:
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    sys.modules["common_util"].get_filename = lambda p: p
    sys.modules["tqdm"].tqdm = lambda x, **k: x
    sys.modules["imgaug"].augmenters = sys.modules["imgaug.augmenters"]
    sys.modules["imgaug"].augmentables = sys.modules["imgaug.augmentables"]
    sys.modules["imgaug.augmentables"].segmaps = sys.modules["imgaug.augmentables.segmaps"]
    sys.modules["imgaug.augmentables.segmaps"].SegmentationMapsOnImage = object
    sys.modules["matplotlib"].cm = sys.modules["matplotlib.cm"]
    import test_util2d as T2                                    # /root/reference/code/test_util2d.py
    return T2


def _net_params(K, C):
    a = [1.2 + 0.4 * k for k in range(K)]
    b = [-0.4 + 0.3 * k for k in range(K)]
    ch = [k % C for k in range(K)]
    return a, b, ch


def gen_sw(T2):
    from tests.helpers import AffinePickNet
    zeros = torch.zeros

    def zeros_cpu(*a, **kw):
        if kw.get("device") == "cuda":
            kw["device"] = "cpu"
        return zeros(*a, **kw)

    out = {}
    for key, (K, shp, orig, patch, stride) in SW.items():
        torch.manual_seed(len(key) + 40)
        image = torch.randn(*shp) * 2.0
        a, b, ch = _net_params(K, shp[1])
        net = AffinePickNet(a, b, ch)
        torch.zeros = zeros_cpu
        try:
            hard, soft = T2.test_single_batch(net, image, orig, patch, stride, "fundus", K, "segtran")
        finally:
            torch.zeros = zeros
        out[key] = dict(K=K, image=image, orig=orig, patch=patch, stride=stride, a=a, b=b, ch=ch, hard=hard.clone(),
                        soft=soft.clone())
        print("sw", key, tuple(hard.shape), hard.dtype, float(soft.mean()))
    return out


def _pred(B, H, W, seed, h, w):
    """a soft prediction at h x w for fundus_like_gt(B, H, W, seed): the same ellipses with jittered radii, noised"""
    return E.soft_from_gt(E.fundus_like_gt(B, H, W, seed, jitter=0.3, jitter_seed=seed + 100), h, w, seed=seed + 200)


def _metric_cases():
    cases = {}
    cases["ellipse"] = dict(K=3, pred=_pred(3, 96, 80, 51, 48, 40), gt=E.fundus_like_gt(3, 96, 80, 51))
    cases["same_size"] = dict(K=3, pred=_pred(2, 40, 36, 53, 40, 36), gt=E.fundus_like_gt(2, 40, 36, 53))
    gt = E.fundus_like_gt(2, 50, 60, 55)[:, 1:3].clone()                  # polyp-like: background + one class
    gt[:, 0] = 1 - gt[:, 1]
    pred = _pred(2, 50, 60, 55, 25, 30)[:, 1:3].clone()
    cases["polyp"] = dict(K=2, pred=pred, gt=gt)
    gt = E.fundus_like_gt(3, 64, 56, 57)
    pred = _pred(3, 64, 56, 57, 32, 28)
    pred[0, 2] *= 0.45                                                    # image 0: the prediction has no cup
    gt[1, 1] = 0                                                          # image 1: the ground truth has no disc
    gt[1, 0] = 1 - gt[1, 2]
    gt[2, 2] = 0                                                          # image 2: cup empty in both (Dice 1)
    gt[2, 0] = 1 - gt[2, 1]
    pred[2, 2] *= 0.45
    cases["edges"] = dict(K=3, pred=pred, gt=gt)
    g1, g2 = E.fundus_like_gt(1, 72, 64, 59)[0], E.fundus_like_gt(1, 48, 52, 60)[0]
    cases["list_two_sizes"] = dict(K=3, pred=[_pred(1, 72, 64, 59, 36, 32)[0], _pred(1, 48, 52, 60, 48, 52)[0]],
                                   gt=[g1, g2])
    return cases


def gen_metric(T2):
    out = {}
    for key, c in _metric_cases().items():
        metric = {}
        for vcdr in ((False, True) if c["K"] >= 3 else (False,)):
            metric[vcdr] = torch.from_numpy(T2.calc_batch_metric(c["pred"], c["gt"], c["K"], do_calc_vcdr_error=vcdr))
        as_u8 = (lambda g: [t.to(torch.uint8) for t in g]) if isinstance(c["gt"], list) else (lambda g: g.to(torch.uint8))
        out[key] = dict(K=c["K"], pred=c["pred"], gt=as_u8(c["gt"]), metric=metric)
        print("metric", key, {k: v.tolist() for k, v in metric.items()})
    return out


def main():
    torch.set_num_threads(4)
    T2 = _ref_util2d()
    fx = dict(kind="eval2d", sw=gen_sw(T2), metric=gen_metric(T2))
    torch.save(fx, os.path.join(OUT, "eval2d.pt"))
    print("wrote", os.path.join(OUT, "eval2d.pt"), os.path.getsize(os.path.join(OUT, "eval2d.pt")), "bytes")


if __name__ == "__main__":
    main()
