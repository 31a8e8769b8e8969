"""Generate tests/golden/metrics_percase.pt and tests/golden/metrics_fullsize.pt (build container only: reads the reference).

TEST INFRASTRUCTURE ONLY.  Run:  python -m oracle.gen_metric_golden
(a) metrics_percase.pt: the REAL test_util3d.calculate_metric_percase (code/test_util3d.py:186-215), with medpy.metric.binary
    stubbed by the restatement in oracle/metric_oracle.py (medpy is not installed; the stubs of gen_golden.gen_infer make
    the module importable), on small seeded cases: a BraTS [4,...] float map, empty pred / empty gt / both empty, a soft
    map with values in (0,1) (the uint8 truncation), and a non-BraTS [H,W,D] long map whose [cls] is a 2-D slice.
(b) metrics_fullsize.pt: 240x240x155, K = 4 cases from metric_oracle.brats_like_case: the seeds, the sha256 of each
    generated volume and the restatement's metrics with hd95 in the hd column (no volumes are stored).
"""
from __future__ import annotations

import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import metric_oracle as M                   # noqa: E402
from oracle import ref_import as R                      # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

FULLSIZE = [dict(seed=101, empty=None), dict(seed=202, empty=("pred", 2)), dict(seed=303, empty=("gt", 1))]


def _ref_percase():
    R.load()
    for name in ("h5py", "nibabel", "medpy", "medpy.metric", "common_util", "tqdm"):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    binary = types.ModuleType("medpy.metric.binary")
    for fn in ("dc", "jc", "asd", "assd", "hd", "hd95"):
        setattr(binary, fn, getattr(M, fn))
    sys.modules["medpy.metric"].binary = binary
    sys.modules["medpy"].metric = sys.modules["medpy.metric"]
    sys.modules["common_util"].get_filename = lambda p: p
    sys.modules["tqdm"].tqdm = lambda x, **k: x
    import test_util3d as T3                                    # /root/reference/code/test_util3d.py
    return T3.calculate_metric_percase


def gen_percase():
    ref = _ref_percase()
    cases = {}
    shape = (24, 20, 16)
    p, g = M.brats_like_case(7, shape, flip_p=2e-3)
    cases["brats"] = dict(pred=p, gt=g, K=4, kind="float")
    p, g = M.brats_like_case(8, shape, flip_p=2e-3)
    p[1].zero_()                                                # class 1: empty prediction
    g[2].zero_()                                                # class 2: empty ground truth
    p[3].zero_()
    g[3].zero_()                                                # class 3: both empty
    cases["empty"] = dict(pred=p, gt=g, K=4, kind="float")
    gen = torch.Generator().manual_seed(9)
    p, g = M.brats_like_case(9, (12, 10, 9), flip_p=1e-2)
    soft = p.float() * (1.0 + torch.rand(p.shape, generator=gen)) \
        + (1 - p.float()) * torch.rand(p.shape, generator=gen) * 0.999    # (0,1) -> 0, [1,2) -> 1 under astype(uint8)
    cases["soft"] = dict(pred=soft, gt=g, K=4, kind="soft")
    lab_p = torch.randint(0, 3, (10, 14, 12), generator=gen)
    lab_g = torch.randint(0, 3, (10, 14, 12), generator=gen)
    lab_p[1, 0, :4] = 256                                       # wraps to 0 under astype(uint8)
    lab_p[2, 3, 5] = 257                                        # wraps to 1
    cases["argmax"] = dict(pred=lab_p, gt=lab_g, K=3, kind="long")
    out = {}
    for key, c in cases.items():
        pred = c["pred"].float() if c["kind"] == "float" else c["pred"]
        gt = c["gt"].float() if c["kind"] in ("float", "soft") else c["gt"]
        metric, valid = ref(pred, gt, c["K"])
        stored_pred = c["pred"] if c["kind"] == "soft" else c["pred"].to(torch.int16 if c["kind"] == "long" else torch.uint8)
        stored_gt = c["gt"].to(torch.int16 if c["kind"] == "long" else torch.uint8)
        out[key] = dict(pred=stored_pred, gt=stored_gt, K=c["K"], kind=c["kind"], metric=torch.from_numpy(metric),
                        valid=torch.from_numpy(valid))
        print("percase", key, metric.tolist(), valid.tolist())
    torch.save(dict(kind="metrics_percase", cases=out), os.path.join(OUT, "metrics_percase.pt"))


def gen_fullsize():
    out = []
    for c in FULLSIZE:
        p, g = M.brats_like_case(c["seed"], empty=c["empty"])
        metric, valid = M.calculate_metric_percase(p, g, 4, hd95_on=True)
        out.append(dict(seed=c["seed"], empty=c["empty"], shape=(240, 240, 155), K=4, sha_pred=M.sha256(p),
                        sha_gt=M.sha256(g), metric=torch.from_numpy(metric), valid=torch.from_numpy(valid)))
        print("fullsize", c, metric.tolist())
    torch.save(dict(kind="metrics_fullsize", cases=out), os.path.join(OUT, "metrics_fullsize.pt"))


if __name__ == "__main__":
    torch.set_num_threads(4)
    gen_percase()
    if len(sys.argv) < 2 or sys.argv[1] != "percase":
        gen_fullsize()
