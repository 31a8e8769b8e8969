"""Restatement of the evaluation metrics (CPU, checker only): medpy 0.4's medpy/metric/binary.py functions dc, jc, asd,
assd, hd and hd95 (unit spacing, connectivity 1) with scipy.ndimage and numpy, the reference's
code/test_util3d.py:186-215 calculate_metric_percase, a pure-torch brute-force definition of the same quantities, and
seeded generators of test volumes (torch's CPU generator, elementwise float64 arithmetic only, so a seed gives the
same bytes on every machine).

scipy is imported inside the functions that need it: the generators and the brute force run without it.
"""
from __future__ import annotations

import hashlib

import numpy as np
import torch
import torch.nn.functional as F


# ---- medpy.metric.binary, restated ------------------------------------------------------------------------------
def dc(result, reference):
    result = np.atleast_1d(np.asarray(result).astype(bool))
    reference = np.atleast_1d(np.asarray(reference).astype(bool))
    # int(): medpy wrote this for count_nonzero returning a Python int, whose division by zero raises and gives 0.0;
    # numpy 2's numpy.int64 would give nan instead
    intersection = int(np.count_nonzero(result & reference))
    size_i1 = int(np.count_nonzero(result))
    size_i2 = int(np.count_nonzero(reference))
    try:
        return 2. * intersection / float(size_i1 + size_i2)
    except ZeroDivisionError:
        return 0.0


def jc(result, reference):
    result = np.atleast_1d(np.asarray(result).astype(bool))
    reference = np.atleast_1d(np.asarray(reference).astype(bool))
    intersection = np.count_nonzero(result & reference)
    union = np.count_nonzero(result | reference)
    return float(intersection) / float(union)


def surface_distances(result, reference):
    """medpy's __surface_distances with voxelspacing=None, connectivity=1."""
    from scipy import ndimage
    result = np.atleast_1d(np.asarray(result).astype(bool))
    reference = np.atleast_1d(np.asarray(reference).astype(bool))
    footprint = ndimage.generate_binary_structure(result.ndim, 1)
    if 0 == np.count_nonzero(result):
        raise RuntimeError('The first supplied array does not contain any binary object.')
    if 0 == np.count_nonzero(reference):
        raise RuntimeError('The second supplied array does not contain any binary object.')
    result_border = result ^ ndimage.binary_erosion(result, structure=footprint, iterations=1)
    reference_border = reference ^ ndimage.binary_erosion(reference, structure=footprint, iterations=1)
    dt = ndimage.distance_transform_edt(~reference_border, sampling=None)
    return dt[result_border]


def asd(result, reference):
    return surface_distances(result, reference).mean()


def assd(result, reference):
    return np.mean((asd(result, reference), asd(reference, result)))


def hd(result, reference):
    return max(surface_distances(result, reference).max(), surface_distances(reference, result).max())


def hd95(result, reference):
    return np.percentile(np.hstack((surface_distances(result, reference), surface_distances(reference, result))), 95)


def calculate_metric_percase(allcls_pred, allcls_gt, num_classes, hd95_on=False):
    """test_util3d.calculate_metric_percase on CPU tensors or arrays; hd95_on=True fills the hd column with hd95."""
    allcls_metric = np.zeros((num_classes - 1, 4))
    allcls_metric_valid = np.ones((num_classes - 1, 4))
    pred_np = allcls_pred.numpy() if isinstance(allcls_pred, torch.Tensor) else np.asarray(allcls_pred)
    gt_np = allcls_gt.numpy() if isinstance(allcls_gt, torch.Tensor) else np.asarray(allcls_gt)
    for cls in range(1, num_classes):
        pred = pred_np[cls].astype(np.uint8)
        gt = gt_np[cls].astype(np.uint8)
        dice = dc(pred, gt)
        if gt.sum() > 0:
            jac = jc(pred, gt)
        else:
            jac = 0
            allcls_metric_valid[cls - 1, 1] = 0
        if pred.sum() > 0 and gt.sum() > 0:
            hdv = hd95(pred, gt) if hd95_on else 0
            asdv = asd(pred, gt)
        else:
            hdv = 0
            asdv = 0
            allcls_metric_valid[cls - 1, 2] = 0
            allcls_metric_valid[cls - 1, 3] = 0
        allcls_metric[cls - 1] = [dice, jac, hdv, asdv]
    return allcls_metric, allcls_metric_valid


# ---- brute-force definition (pure torch) --------------------------------------------------------------------------
def brute_border(x: torch.Tensor) -> torch.Tensor:
    """Foreground voxels with a background (or outside-the-volume) voxel among their 2*ndim axis neighbours."""
    x = x.bool()
    p = F.pad(x.to(torch.uint8)[None, None], (1, 1) * x.dim(), value=0)[0, 0].bool()
    inner = torch.ones_like(x)
    for ax in range(x.dim()):
        for s in (0, 2):                                   # the neighbour before / after along this axis
            sl = [slice(1, 1 + n) for n in x.shape]
            sl[ax] = slice(s, s + x.shape[ax])
            inner &= p[tuple(sl)]
    return x & ~inner


def brute_sq_distances(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Integer squared distance from every border voxel of a to the nearest border voxel of b (int64)."""
    pa = brute_border(a).nonzero().long()
    pb = brute_border(b).nonzero().long()
    d2 = ((pa[:, None, :] - pb[None, :, :]) ** 2).sum(-1)
    return d2.min(1).values


def brute_percentile95(vals: torch.Tensor) -> float:
    """numpy's linear percentile, restated: vi = (n-1)*0.95, lerp between the order statistics floor(vi), floor(vi)+1."""
    s = torch.sort(vals.double()).values.tolist()
    n = len(s)
    vi = (n - 1) * 0.95
    lo = int(np.floor(vi))
    g = vi - lo
    a, b = s[lo], s[min(lo + 1, n - 1)]
    return b - (b - a) * (1 - g) if g >= 0.5 else a + (b - a) * g


def brute_metrics(a: torch.Tensor, b: torch.Tensor) -> dict:
    """dc, jc and (both masks non-empty) asd, assd, hd, hd95 of result a against reference b."""
    a, b = a.bool(), b.bool()
    inter, na, nb, union = int((a & b).sum()), int(a.sum()), int(b.sum()), int((a | b).sum())
    out = dict(dc=2. * inter / float(na + nb) if na + nb else 0.0, jc=float(inter) / float(union) if union else None)
    if na and nb:
        # numpy's sqrt is correctly rounded; torch's CPU sqrt of float64 can be one ulp off
        dab = torch.from_numpy(np.sqrt(brute_sq_distances(a, b).numpy().astype(np.float64)))
        dba = torch.from_numpy(np.sqrt(brute_sq_distances(b, a).numpy().astype(np.float64)))
        out.update(asd=float(dab.mean()), asd_ba=float(dba.mean()), hd=float(max(dab.max(), dba.max())),
                   hd95=brute_percentile95(torch.cat([dab, dba])))
        out["assd"] = float(np.mean((out["asd"], out["asd_ba"])))
    return out


# ---- seeded volumes -------------------------------------------------------------------------------------------------
def _ellipsoid(shape, centre, radii):
    axes = [torch.arange(n, dtype=torch.float64) for n in shape]
    acc = None
    for ax, (x, c, r) in enumerate(zip(axes, centre, radii)):
        t = (x - c) / r
        t = (t * t).reshape([-1 if a == ax else 1 for a in range(len(shape))])
        acc = t if acc is None else acc + t
    return acc <= 1.0


def brats_like_case(seed: int, shape=(240, 240, 155), K: int = 4, empty=None, flip_p=2e-5):
    """(pred, gt) uint8 [K, *shape]: class k >= 1 of gt is one or two ellipsoids with seeded centres and radii, pred
    jitters them and flips sparse voxels of the whole volume; class K-1's gt ellipsoid is centred on the volume's first
    face, so it touches the boundary.  empty=("pred" | "gt", k) leaves that class empty on that side.  Class 0 is the
    background (no class fired), as in the BraTS maps."""
    g = torch.Generator().manual_seed(int(seed))
    n = torch.tensor(shape, dtype=torch.float64)
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)         # noqa: E731
    pred = torch.zeros((K,) + tuple(shape), dtype=torch.uint8)
    gt = torch.zeros_like(pred)
    for k in range(1, K):
        for e in range(1 + (k % 2)):
            c = n * (0.3 + 0.4 * u(3))
            r = n * (0.06 + 0.12 * u(3))
            if k == K - 1 and e == 0:
                c[0] = 0.0
            cp = c + (u(3) - 0.5) * 0.2 * r
            rp = r * (0.85 + 0.3 * u(3))
            gt[k] |= _ellipsoid(shape, c.tolist(), r.tolist()).to(torch.uint8)
            pred[k] |= _ellipsoid(shape, cp.tolist(), rp.tolist()).to(torch.uint8)
        flip = (torch.rand(tuple(shape), generator=g) < flip_p).to(torch.uint8)
        pred[k] ^= flip
    if empty is not None:
        side, k = empty
        (pred if side == "pred" else gt)[k].zero_()
    pred[0] = (pred[1:].sum(0) == 0).to(torch.uint8)
    gt[0] = (gt[1:].sum(0) == 0).to(torch.uint8)
    return pred, gt


def sha256(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def small_volumes(seed: int = 0):
    """Random (result, reference) bool pairs, 2-D and 3-D: odd and prime extents, extents of 1, single-voxel objects,
    all-foreground volumes, objects touching the boundary, sparse and dense noise."""
    g = torch.Generator().manual_seed(seed)
    shapes = [(7, 11), (13, 1), (1, 17), (5, 5), (29, 23), (3, 7, 5), (1, 9, 11), (7, 1, 13), (11, 13, 1), (9, 8, 7),
              (17, 19, 13), (1, 1, 31)]
    cases = []
    for sh in shapes:
        for p in (0.05, 0.3, 0.7):
            a = torch.rand(sh, generator=g) < p
            b = torch.rand(sh, generator=g) < p
            a.view(-1)[0] = True                                  # a voxel on the boundary: never empty
            b.view(-1)[-1] = True
            cases.append((a, b))
        one_a = torch.zeros(sh, dtype=torch.bool)
        one_b = torch.zeros(sh, dtype=torch.bool)
        one_a.view(-1)[int(torch.randint(one_a.numel(), (1,), generator=g))] = True
        one_b.view(-1)[int(torch.randint(one_b.numel(), (1,), generator=g))] = True
        cases.append((one_a, one_b))                              # single-voxel objects
        cases.append((torch.ones(sh, dtype=torch.bool), one_b))   # all foreground against a single voxel
        cases.append((torch.ones(sh, dtype=torch.bool), torch.ones(sh, dtype=torch.bool)))
    return cases
