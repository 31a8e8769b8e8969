"""Evaluation metrics on the GPU: a drop-in for the reference's ``test_util3d.calculate_metric_percase``
(code/test_util3d.py:186-215) and medpy 0.4's ``dc, jc, hd, hd95, asd, assd`` (medpy/metric/binary.py) on CUDA tensors,
with unit voxel spacing and connectivity 1; and for the 2-D evaluation, ``test_util2d.calc_batch_metric`` and the
unbatched ``utils/losses.calc_vcdr`` (per-image Dice and vertical cup-to-disc ratio, csrc/sx_eval2d.cu).

Every distance is sqrt of an exact integer squared distance, so the library's kernels (csrc/sx_metrics.cu) compute
the same dc, jc, hd and hd95 as medpy bit for bit, and asd to the last bits of an fp64 sum in another order.  All
medpy-style functions go through ``_case_metrics``: one fixed sequence of launches for all classes of a case, one
device-to-host copy.  The 2-D functions go through ``_eval2d_counts``: one launch per batch, one device-to-host copy.
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


# ------------------------------------------------------------------------------------------------
# 2-D per-image evaluation: drop-ins for test_util2d.calc_batch_metric / calc_dice (code/test_util2d.py:229-265) and the
# unbatched branch of utils/losses.calc_vcdr (:76-127), from the integer counts of sx_eval2d_counts (csrc/sx_eval2d.cu)
# ------------------------------------------------------------------------------------------------
_ROWS = 8                     # row slots per image: {pred, gt} x {disc, cup} x {last row + 1, H - first row}


def _eval2d_ld(K: int) -> int:
    return 3 * (K - 1) + _ROWS + 1


def _eval2d_counts(preds, gts, K: int) -> np.ndarray:
    """preds: a [B,K',h,w] CUDA tensor or a list of [K',h,w] ones (None: ground-truth part only); gts likewise, with
    K', h, w free per image in a list.  -> int64 [B, 3(K-1) + 9] counts of the first K classes, one device-to-host copy."""
    B = len(gts)
    if preds is not None and len(preds) != B:
        raise ValueError("calc_batch_metric: %d predictions for %d ground truths" % (len(preds), B))
    if B == 0:
        return np.zeros((0, _eval2d_ld(K)), dtype=np.int64)
    if torch.is_tensor(gts) and (preds is None or torch.is_tensor(preds)):
        groups = [(preds, gts)]                                     # one shape: the whole batch in one launch
    else:                                                           # images of different sizes: one launch each
        groups = [(None if preds is None else preds[b].unsqueeze(0), gts[b].unsqueeze(0)) for b in range(B)]
    for p, g in groups:
        ops._req_cuda(p, g)
        if g.dim() != 4 or g.shape[1] < K or (p is not None and (p.dim() != 4 or p.shape[1] < K)):
            raise ValueError("calc_batch_metric: need [C,H,W] maps of at least %d classes, got %s and %s"
                             % (K, None if p is None else tuple(p.shape[1:]), tuple(g.shape[1:])))
    counts = torch.zeros((B, _eval2d_ld(K)), device=groups[0][1].device, dtype=torch.int32)
    st = ops._stream()
    b0 = 0
    for p, g in groups:
        g = g[:, :K].float().contiguous()
        h = w = 0
        if p is not None:
            p = p[:, :K].float().contiguous()
            h, w = p.shape[2:]
        n = g.shape[0]
        L.call("sx_eval2d_counts", ops._ptr(p), n, K, h, w, g.data_ptr(), g.shape[2], g.shape[3], counts[b0].data_ptr(),
               st)
        b0 += n
    return counts.cpu().numpy().astype(np.int64)


def _vcdr(rows: np.ndarray, H: int) -> np.float32:
    """calc_vcdr (losses.py:102-127) of one mask from its four row slots [disc last+1, disc H-first, cup last+1,
    cup H-first]: fp32 cup_len / (disc_len + 1e-4) with len = last - first - 1; -1 without a disc, 0 without a cup."""
    if rows[0] == 0:
        return np.float32(-1.)
    disc_len = int(rows[0] - 1) - int(H - rows[1]) - 1
    if rows[2] == 0:
        return np.float32(0.)
    cup_len = int(rows[2] - 1) - int(H - rows[3]) - 1
    return np.float32(cup_len) / (np.float32(disc_len) + np.float32(1e-4))


def _batch_values(counts: np.ndarray, K: int, heights, do_calc_vcdr_error: bool) -> np.ndarray:
    """calc_batch_metric's array from the counts of sx_eval2d_counts, in the reference's fp32 operation order.
    heights: the ground-truth height of each image."""
    B = counts.shape[0]
    nc = K - 1
    bad = counts[:, 3 * nc + _ROWS]
    if bad.any():
        raise ValueError("calc_batch_metric: the ground truth must be binary (0/1); %d values of classes 1..%d are not"
                         % (int(bad.sum()), nc))
    out = np.zeros((B, nc + int(bool(do_calc_vcdr_error))))
    eps = np.float32(1e-5)
    for b in range(B):
        for c in range(nc):
            inter, p, g = (np.float32(v) for v in counts[b, 3 * c:3 * c + 3])
            out[b, c] = (np.float32(2) * inter + eps) / ((p + g) + eps)          # calc_dice, test_util2d.py:229-236
        if do_calc_vcdr_error:
            r = counts[b, 3 * nc:3 * nc + _ROWS]
            out[b, nc] = np.abs(_vcdr(r[4:], heights[b]) - _vcdr(r[:4], heights[b]))
    return out


def _require_vcdr_classes(K: int):
    if K < 3:
        raise ValueError("vCDR needs the disc (class 1) and cup (class 2) channels: num_classes >= 3, got %d" % K)


def calc_batch_metric(BC_pred_soft, BC_gt, num_classes, do_calc_vcdr_error=False):
    """Drop-in for test_util2d.calc_batch_metric: per image, the soft prediction bilinearly resized to its ground truth's
    size and hardened at 0.5 (harden_segmap2d), the Dice of each class 1..K-1 ((2|P and G| + 1e-5) / (|P| + |G| + 1e-5)
    in fp32) and, with do_calc_vcdr_error, |vCDR(gt) - vCDR(pred)|.  BC_pred_soft / BC_gt: [B,K,h,w] / [B,K,H,W] CUDA
    tensors, or lists of [K,h,w] / [K,H,W] ones of per-image sizes.  The ground truth must be binary (every
    mask_prepred_mapping_func gives 0/1): ValueError otherwise.  One kernel launch per batch (per image for lists) and one
    device-to-host copy.  -> float64 numpy [B, K-1+do_calc_vcdr_error], bit-identical to the reference for the same
    hard masks."""
    K = int(num_classes)
    if do_calc_vcdr_error:
        _require_vcdr_classes(K)
    if K < 2:
        raise ValueError("calc_batch_metric: num_classes must be >= 2, got %d" % K)
    counts = _eval2d_counts(BC_pred_soft, BC_gt, K)
    heights = [int(g.shape[-2]) for g in BC_gt]
    return _batch_values(counts, K, heights, do_calc_vcdr_error)


def calc_vcdr(mask):
    """Drop-in for utils/losses.calc_vcdr on one [C,H,W] mask (C >= 3; classes 1: disc, 2: cup; occupied = >= 0.5):
    the vertical cup-to-disc ratio as a 0-dim fp32 tensor on the mask's device (-1 without a disc, 0 without a cup)."""
    ops._req_cuda(mask)
    if mask.dim() != 3:
        raise ValueError("calc_vcdr: one [C,H,W] mask expected (the batched form is not implemented), got %s"
                         % (tuple(mask.shape),))
    _require_vcdr_classes(mask.shape[0])
    counts = _eval2d_counts(None, mask[:3].unsqueeze(0), 3)
    rows = counts[0, 6:6 + _ROWS]
    return torch.tensor(_vcdr(rows[4:], int(mask.shape[1])), device=mask.device)
