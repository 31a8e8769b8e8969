"""Evaluation metrics on the GPU: a drop-in for the reference's ``test_util3d.calculate_metric_percase``
(code/test_util3d.py:186-215) and medpy 0.4's ``dc, jc, hd, hd95, asd, assd`` (medpy/metric/binary.py) on CUDA tensors,
with unit voxel spacing and connectivity 1.

Every distance is sqrt of an exact integer squared distance, so the library's kernels (csrc/sx_metrics.cu) compute
the same dc, jc, hd and hd95 as medpy bit for bit, and asd to the last bits of an fp64 sum in another order.  All
functions go through ``_case_metrics``: one fixed sequence of launches for all classes of a case, one device-to-host copy.
No CPU fallback: the masks must live on the GPU.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib as L
from . import ops

_LDO = 12          # per class: 4 int64 counts, then the 8 fp64 statistics of sx_surface_stats


def _case_metrics(A: torch.Tensor, B: torch.Tensor, ndim: int) -> np.ndarray:
    """A, B: uint8 [K, *spatial] CUDA masks (non-zero = foreground), len(spatial) == ndim.
    -> float64 [K, 12] on the host: columns 0-3 the int64 counts |A|, |B|, |A and B|, |A or B| (bit views), then
    n(A->B), n(B->A), asd(A->B), asd(B->A), max(A->B), max(B->A), hd95 of both directions, n of both."""
    K = A.shape[0]
    n0, n1, n2 = ((1,) + tuple(A.shape[1:])) if ndim == 2 else tuple(A.shape[1:])
    V = n0 * n1 * n2
    nbins = (n0 - 1) ** 2 + (n1 - 1) ** 2 + (n2 - 1) ** 2 + 1
    dev, st = A.device, ops._stream()
    A, B = A.contiguous(), B.contiguous()
    res = torch.empty(K, _LDO, device=dev, dtype=torch.float64)
    L.call("sx_mask_counts", A.data_ptr(), B.data_ptr(), K, V, res.data_ptr(), _LDO, st)
    bA = torch.empty(K, V, device=dev, dtype=torch.uint8)
    bB = torch.empty(K, V, device=dev, dtype=torch.uint8)
    L.call("sx_surface", A.data_ptr(), K, ndim, n0, n1, n2, bA.data_ptr(), st)
    L.call("sx_surface", B.data_ptr(), K, ndim, n0, n1, n2, bB.data_ptr(), st)
    dist = torch.empty(K, V, device=dev, dtype=torch.int32)
    hist = torch.empty(K, 2, nbins, device=dev, dtype=torch.int32)        # read as uint32 by the kernels
    for d, (src, dst) in enumerate(((bA, bB), (bB, bA))):                  # medpy's __surface_distances(src, dst)
        L.call("sx_edt_sq", dst.data_ptr(), K, n0, n1, n2, dist.data_ptr(), st)
        L.call("sx_surface_hist", src.data_ptr(), dist.data_ptr(), K, V, nbins, hist[:, d].data_ptr(), 2 * nbins, st)
    L.call("sx_surface_stats", hist.data_ptr(), K, nbins, 2 * nbins, res[:, 4:].data_ptr(), _LDO, st)
    return res.cpu().numpy()


def _counts(h: np.ndarray) -> np.ndarray:
    return h[:, :4].copy().view(np.int64)


def _dc(c) -> float:
    inter, size = int(c[2]), int(c[0]) + int(c[1])
    return 2. * inter / float(size) if size else 0.0


def _jc(c) -> float:
    return float(int(c[2])) / float(int(c[3]))


def _check_args(voxelspacing, connectivity):
    if voxelspacing is not None:
        raise NotImplementedError("segtran_b200.metrics: only unit voxel spacing is implemented (voxelspacing=None); "
                                  "anisotropic distances are not square roots of integers")
    if connectivity != 1:
        raise NotImplementedError("segtran_b200.metrics: only connectivity=1 (the axis-neighbour cross) is implemented, "
                                  "got %r" % (connectivity,))


def _pair(result: torch.Tensor, reference: torch.Tensor, voxelspacing, connectivity):
    """medpy's operand handling for one pair: bool cast, ndim 2 or 3, same shape -> one row of _case_metrics."""
    _check_args(voxelspacing, connectivity)
    ops._req_cuda(result, reference)
    if result.dim() not in (2, 3):
        raise ValueError("segtran_b200.metrics: masks must have 2 or 3 dimensions, got %d" % result.dim())
    if result.shape != reference.shape:
        raise ValueError("segtran_b200.metrics: result %s and reference %s differ in shape"
                         % (tuple(result.shape), tuple(reference.shape)))
    a = result.to(torch.bool).view(torch.uint8).unsqueeze(0)
    b = reference.to(torch.bool).view(torch.uint8).unsqueeze(0)
    h = _case_metrics(a, b, result.dim())
    return _counts(h)[0], h[0, 4:]


def _require_objects(c):
    if c[0] == 0:
        raise RuntimeError("The first supplied array does not contain any binary object.")
    if c[1] == 0:
        raise RuntimeError("The second supplied array does not contain any binary object.")


def dc(result, reference, voxelspacing=None, connectivity=1) -> float:
    """Dice coefficient 2|A and B| / (|A| + |B|), 0.0 when both are empty (medpy.metric.binary.dc)."""
    c, _ = _pair(result, reference, voxelspacing, connectivity)
    return _dc(c)


def jc(result, reference, voxelspacing=None, connectivity=1) -> float:
    """Jaccard coefficient |A and B| / |A or B| (medpy.metric.binary.jc)."""
    c, _ = _pair(result, reference, voxelspacing, connectivity)
    return _jc(c)


def asd(result, reference, voxelspacing=None, connectivity=1) -> float:
    """Mean distance from result's surface voxels to reference's surface (one direction; medpy.metric.binary.asd).
    RuntimeError when either mask is empty."""
    c, s = _pair(result, reference, voxelspacing, connectivity)
    _require_objects(c)
    return float(s[2])


def assd(result, reference, voxelspacing=None, connectivity=1) -> float:
    """Mean of asd(result, reference) and asd(reference, result) (medpy.metric.binary.assd)."""
    c, s = _pair(result, reference, voxelspacing, connectivity)
    _require_objects(c)
    return float(np.mean((s[2], s[3])))


def hd(result, reference, voxelspacing=None, connectivity=1) -> float:
    """Hausdorff distance: the maximum surface distance over both directions (medpy.metric.binary.hd)."""
    c, s = _pair(result, reference, voxelspacing, connectivity)
    _require_objects(c)
    return float(max(s[4], s[5]))


def hd95(result, reference, voxelspacing=None, connectivity=1) -> float:
    """95th percentile (numpy's linear method) of the surface distances of both directions together
    (medpy.metric.binary.hd95)."""
    c, s = _pair(result, reference, voxelspacing, connectivity)
    _require_objects(c)
    return float(s[6])


def calculate_metric_percase(allcls_pred, allcls_gt, num_classes, hd95=False):
    """Drop-in for test_util3d.calculate_metric_percase: for each class 1..num_classes-1, [dice, jc, hd, asd] of
    allcls_pred[cls] against allcls_gt[cls] after the reference's astype(uint8), and the validity flags.
    allcls_pred / allcls_gt: CUDA tensors (the float [K,H,W,D] BraTS maps, or the [H,W,D] argmax maps, whose [cls] is a
    2-D slice, as in the reference).  hd95=False reproduces the reference, whose hd column is 0; hd95=True fills that
    column with the HD95 of each class whose masks are both non-empty (the valid flags stay the reference's).
    -> (metric [K-1, 4] float64, valid [K-1, 4] float64) numpy arrays."""
    K = int(num_classes)
    ops._req_cuda(allcls_pred, allcls_gt)
    metric = np.zeros((K - 1, 4))
    valid = np.ones((K - 1, 4))
    if K < 2:
        return metric, valid
    ndim = allcls_pred.dim() - 1
    if ndim not in (2, 3):
        raise ValueError("calculate_metric_percase: per-class masks must have 2 or 3 dimensions, got %d" % ndim)
    if allcls_pred.shape[1:] != allcls_gt.shape[1:] or min(allcls_pred.shape[0], allcls_gt.shape[0]) < K:
        raise ValueError("calculate_metric_percase: need %d classes of one shape, got %s and %s"
                         % (K, tuple(allcls_pred.shape), tuple(allcls_gt.shape)))
    pred = allcls_pred[1:K].to(torch.uint8)
    gt = allcls_gt[1:K].to(torch.uint8)
    h = _case_metrics(pred, gt, ndim)
    counts = _counts(h)
    for i in range(K - 1):
        c, s = counts[i], h[i, 4:]
        dice, jac, hdv, asdv = _dc(c), 0, 0, 0
        if c[1] > 0:
            jac = _jc(c)
        else:
            valid[i, 1] = 0
        if c[0] > 0 and c[1] > 0:
            hdv = s[6] if hd95 else 0
            asdv = s[2]
        else:
            valid[i, 2] = 0
            valid[i, 3] = 0
        metric[i] = [dice, jac, hdv, asdv]
    return metric, valid
