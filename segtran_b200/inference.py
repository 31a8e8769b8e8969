"""Sliding-window inference of a whole volume (SURVEY.md §8 f.4): drop-in for the reference's
``test_util3d.test_single_case`` (code/test_util3d.py:93-184) — same signature, same window enumeration, same padding —
with the per-patch "sigmoid -> accumulate -> count" update and the final "average -> BraTS consistency -> threshold"
running as two library kernels (csrc/sx_infer.cu) and the two tri-linear resizes as the library's per-axis kernels.
``test_single_batch`` is the 2-D counterpart for ``test_util2d.test_single_batch`` (csrc/sx_eval2d.cu), with the score
upsample folded into the accumulating kernel.  No CPU fallback: the images must live on the GPU.

Both take an opt-in ``mirror_axes`` (mirror test-time augmentation, beyond the reference): every window batch is also
predicted mirrored along each non-empty subset of those axes, and the scores, flipped back, are averaged with the
plain ones.  The mirrored windows are gathered straight from the padded image by one kernel (``sx_sw_gather``), and the
accumulating kernels read the scores through reversed indices, so no flipped score map is written.

Both also take an opt-in ``gaussian_sigma_scale`` (Gaussian importance weighting of the overlapping windows, as in
nnU-Net and MONAI's ``mode="gaussian"``): each window adds w * sigmoid(score) and w to the count, with w a separable
Gaussian of the position inside the window, so voxels near a window's centre count more than those at its edges.  The
accumulating kernels apply the weight from per-axis tables that each accumulate call is given (``sx_sw_weights``)."""
from __future__ import annotations

import ctypes
import math
import numbers
from collections.abc import Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib as L
from . import ops


def _resize(x, size):
    """F.interpolate(x, size, mode='bilinear' / 'trilinear', align_corners=False) via the library's per-axis kernels
    (no-op if equal)."""
    if tuple(x.shape[2:]) == tuple(size):
        return x
    return ops.resize_linear(x.float(), tuple(int(s) for s in size))


def _mirror_masks(mirror_axes, ndim, who):
    """The kernels' mirror masks of the 2^k variants of ``mirror_axes`` (distinct spatial axes in [0, ndim)), in variant
    order: variant m mirrors mirror_axes[i] for every bit i set in m, and variant 0 is the identity."""
    if isinstance(mirror_axes, (str, bytes)) or not isinstance(mirror_axes, Sequence):
        raise ValueError("%s: mirror_axes must be a sequence of spatial axes, got %r" % (who, mirror_axes))
    for a in mirror_axes:
        if isinstance(a, bool) or not isinstance(a, numbers.Integral) or not 0 <= a < ndim:
            raise ValueError("%s: mirror axis %r is not one of the spatial axes 0..%d" % (who, a, ndim - 1))
    axes = [int(a) for a in mirror_axes]
    if len(set(axes)) != len(axes):
        raise ValueError("%s: mirror_axes %r repeats an axis" % (who, tuple(mirror_axes)))
    return [sum(1 << a for i, a in enumerate(axes) if m >> i & 1) for m in range(1 << len(axes))]


def _sigma_scale(gaussian_sigma_scale, who):
    """None, or the finite sigma scale s > 0 as a float."""
    s = gaussian_sigma_scale
    if s is None:
        return None
    if isinstance(s, bool) or not isinstance(s, numbers.Real) or not math.isfinite(s) or not s > 0:
        raise ValueError("%s: gaussian_sigma_scale must be None or a finite real number > 0, got %r" % (who, s))
    return float(s)


def gaussian_window_tables(size, sigma_scale):
    """The per-axis weight tables of a window of extent ``size`` = (d_0, d_1, ...), concatenated in axis order as one fp32
    tensor: g(i) = exp(-(i - (d-1)/2)^2 / (2 (s d)^2)) for i = 0..d-1, computed in float64 and divided by its maximum
    over i, then rounded to fp32.  An element's weight is max(g_0(i) * g_1(j) [* g_2(l)], 1e-3), taken in fp32 by the
    accumulating kernels.  The division by the maximum is taken in the exponent (the maximum is at the centre cell(s),
    (i - (d-1)/2)^2 = m with m = 0 or 1/4), so a tiny s cannot make it 0 / 0."""
    out = []
    for d in size:
        sd = sigma_scale * d
        q = (np.arange(d, dtype=np.float64) - (d - 1) / 2.0) ** 2
        out.append(np.exp(-(q - q.min()) / (2.0 * sd * sd)))
    return torch.from_numpy(np.concatenate(out)).float()


def _window_weights(size, sigma_scale, device):
    """(tables, weights): the per-axis tables of the ``size`` window on ``device`` (built once per call) and the
    ``weights`` argument of every accumulate launch, a reference to the sx_sw_weights descriptor that addresses them;
    (None, None) without weighting.  A 2-D window passes no z table."""
    if sigma_scale is None:
        return None, None
    tab = gaussian_window_tables(size, sigma_scale).to(device)
    p, n = tab.data_ptr(), [int(d) for d in size]
    if len(n) == 2:
        desc = L.sx_sw_weights(p, p + 4 * n[0], None, n[0], n[1], 1)
    else:
        desc = L.sx_sw_weights(p, p + 4 * n[0], p + 4 * (n[0] + n[1]), *n)
    return tab, ctypes.byref(desc)


def _tta_image(img, who):
    if img.dtype != torch.float32:
        raise ValueError("%s: mirror_axes needs a float32 image, got %s" % (who, img.dtype))
    return img.contiguous()


def _gather(img, origins, win, mirror):
    """sx_sw_gather: the windows of size ``win`` at ``origins`` of the contiguous fp32 [B,C,*spatial] image, mirrored by
    ``mirror`` (bit a reverses spatial axis a), as [len(origins) * B, C, *win]; a 2-D image is gathered as depth 1."""
    B, C = img.shape[:2]
    spatial = tuple(img.shape[2:]) + (1,) * (5 - img.dim())
    org = [int(v) for o in origins for v in tuple(o) + (0,) * (3 - len(o))]
    out = torch.empty((len(origins) * B, C) + tuple(win), device=img.device, dtype=torch.float32)
    L.call("sx_sw_gather", img.data_ptr(), B, C, *spatial, (ctypes.c_int32 * len(org))(*org), len(origins),
           *(tuple(win) + (1,) * (3 - len(win))), mirror, out.data_ptr(), ops._stream())
    return out


def test_single_case(net, image, orig_patch_size, input_patch_size, batch_size, stride_xy, stride_z, task_name, net_type,
                     num_classes, *, mirror_axes=(), gaussian_sigma_scale=None):
    """image [C,H,W,D] (CUDA) -> (preds_hard, preds_soft), exactly as the reference's function of the same name.

    mirror_axes: distinct axes among 0, 1, 2 (H, W, D).  With k of them, each window batch is predicted 2^k times, on
    flip_m(batch) for every subset m of the axes (the net sees batch_size windows per call, as without them), and the
    scores are flipped back, resized, passed through the sigmoid and accumulated, each variant adding one to the window
    count.  The soft output is the mean over the variants of this function run with the net x -> flip_m(net(flip_m(x))).
    The flip back is read by the accumulating kernel after the resize to the window size; it commutes with the resize up
    to rounding.  The image must be float32 then.  () is the reference's computation.

    gaussian_sigma_scale: None (the reference's flat average) or s > 0: every window, and every mirror variant of it,
    adds w * sigmoid(score) to the soft map and w to the count, with w the Gaussian weight of the position inside the
    orig_patch_size window (gaussian_window_tables; sigma = s times the window's extent along each axis, floored at 1e-3).
    The soft output is then the weighted average.  nnU-Net uses s = 1/8."""
    masks = _mirror_masks(mirror_axes, 3, "test_single_case")
    sigma = _sigma_scale(gaussian_sigma_scale, "test_single_case")
    ops._req_cuda(image)
    C, H, W, D = image.shape
    dx, dy, dz = orig_patch_size
    h_pad, w_pad, d_pad = max(dx - H, 0), max(dy - W, 0), max(dz - D, 0)
    add_pad = (h_pad + w_pad + d_pad) > 0
    hl_pad, hr_pad = h_pad // 2, h_pad - h_pad // 2
    wl_pad, wr_pad = w_pad // 2, w_pad - w_pad // 2
    dl_pad, dr_pad = d_pad // 2, d_pad - d_pad // 2
    if add_pad:
        image = F.pad(image, (dl_pad, dr_pad, wl_pad, wr_pad, hl_pad, hr_pad), mode='constant', value=0)
    C, H2, W2, D2 = image.shape
    sx = math.ceil((H2 - dx) / stride_xy) + 1
    sy = math.ceil((W2 - dy) / stride_xy) + 1
    sz = math.ceil((D2 - dz) / stride_z) + 1
    K = int(num_classes)
    dev = image.device
    preds_soft = torch.zeros((K, H2, W2, D2), device=dev, dtype=torch.float32)
    cnt = torch.zeros((H2, W2, D2), device=dev, dtype=torch.float32)
    st = ops._stream
    img = _tta_image(image, "test_single_case").unsqueeze(0) if len(masks) > 1 else None
    wtab, wts = _window_weights((dx, dy, dz), sigma, dev)      # wtab owns the tables the descriptor points to

    for x in range(sx):
        xs = min(stride_xy * x, H2 - dx)
        yzs_batch, test_patches = [], []
        for y in range(sy):
            ys = min(stride_xy * y, W2 - dy)
            for z in range(sz):
                zs = min(stride_z * z, D2 - dz)
                test_patches.append(image[:, xs:xs + dx, ys:ys + dy, zs:zs + dz])
                yzs_batch.append((ys, zs))
                if len(test_patches) == batch_size or (y == sy - 1 and z == sz - 1):
                    for m in masks:                                  # variants in a fixed order: same bits every run
                        if m == 0:
                            test_batch = _resize(torch.stack(test_patches, dim=0), input_patch_size)
                        else:
                            test_batch = _resize(_gather(img, [(xs,) + yz for yz in yzs_batch], (dx, dy, dz), m),
                                                 input_patch_size)
                        with torch.no_grad():
                            scores_raw = net(test_batch)
                        if net_type == 'unet':
                            scores_raw = scores_raw[1]
                        scores_raw = _resize(scores_raw, orig_patch_size).float().contiguous()
                        for i, (ys_i, zs_i) in enumerate(yzs_batch):   # sequential launches: overlapping windows never race
                            L.call("sx_sw_accumulate", scores_raw[i].data_ptr(), K, dx, dy, dz, preds_soft.data_ptr(),
                                   cnt.data_ptr(), H2, W2, D2, xs, ys_i, zs_i, m, wts, st())
                        del test_batch, scores_raw                     # one variant's batch alive at a time
                    test_patches, yzs_batch = [], []

    brats = task_name == 'brats'
    hard = torch.empty((K, H2, W2, D2) if brats else (H2, W2, D2), device=dev, dtype=torch.float32)
    L.call("sx_sw_finalize", preds_soft.data_ptr(), cnt.data_ptr(), K, H2 * W2 * D2, 1 if brats else 0, hard.data_ptr(), st())
    preds_hard = hard if brats else hard.long()
    if add_pad:
        sl = (slice(hl_pad, hl_pad + H), slice(wl_pad, wl_pad + W), slice(dl_pad, dl_pad + D))
        preds_hard = (preds_hard[(slice(None),) + sl] if brats else preds_hard[sl]).clone()
        preds_soft = preds_soft[(slice(None),) + sl].clone()
    return preds_hard, preds_soft


def test_single_batch(net, image_batch, orig_input_size, patch_size, stride, task_name, num_classes, model_type, *,
                      mirror_axes=(), gaussian_sigma_scale=None):
    """image_batch [B,C,H,W] (CUDA) -> (preds_hard int32 [B,K,H,W], preds_soft fp32 [B,K,H,W]), exactly as the reference's
    test_util2d.test_single_batch (code/test_util2d.py:151-225): zero-pad to orig_input_size, one window per launch in the
    reference's order, each window's scores upsampled, passed through the sigmoid and accumulated by one kernel
    (csrc/sx_eval2d.cu), then average, harden_segmap2d and the crop by another.  task_name is unused, as in the reference.

    mirror_axes: distinct axes among 0, 1 (H, W); as in test_single_case, each window is predicted on flip_m(window) for
    every subset m, and the scores are flipped back (by reversing the upsample's source taps), upsampled and accumulated,
    so the soft output is the mean over the variants of the net x -> flip_m(net(flip_m(x))).  The image must be float32
    then.  () is the reference's computation.

    gaussian_sigma_scale: as in test_single_case, on the orig_input_size window: the weight is applied after the
    upsample, at the window position the upsampled score lands on."""
    masks = _mirror_masks(mirror_axes, 2, "test_single_batch")
    sigma = _sigma_scale(gaussian_sigma_scale, "test_single_batch")
    ops._req_cuda(image_batch)
    B, C, H, W = image_batch.shape
    dx, dy = orig_input_size
    h_pad, w_pad = max(dx - H, 0), max(dy - W, 0)
    add_pad = (h_pad + w_pad) > 0
    hl_pad, hr_pad = h_pad // 2, h_pad - h_pad // 2
    wl_pad, wr_pad = w_pad // 2, w_pad - w_pad // 2
    if add_pad:
        image_batch = F.pad(image_batch, (wl_pad, wr_pad, hl_pad, hr_pad), mode='constant', value=0)
    H2, W2 = image_batch.shape[2:]
    sx = math.ceil((H2 - dx) / stride[0]) + 1
    sy = math.ceil((W2 - dy) / stride[1]) + 1
    K = int(num_classes)
    dev = image_batch.device
    preds = torch.zeros((B, K, H2, W2), device=dev, dtype=torch.float32)
    cnt = torch.zeros((H2, W2), device=dev, dtype=torch.float32)
    st = ops._stream
    img = _tta_image(image_batch, "test_single_batch") if len(masks) > 1 else None
    wtab, wts = _window_weights((dx, dy), sigma, dev)          # wtab owns the tables the descriptor points to

    for x in range(sx):
        xs = min(stride[0] * x, H2 - dx)
        for y in range(sy):
            ys = min(stride[1] * y, W2 - dy)
            for m in masks:                                 # variants in a fixed order: same bits every run
                if m == 0:
                    test_patch = _resize(image_batch[:, :, xs:xs + dx, ys:ys + dy], patch_size)
                else:
                    test_patch = _resize(_gather(img, [(xs, ys)], (dx, dy), m), patch_size)
                with torch.no_grad():
                    scores_raw = net(test_patch)
                if model_type == 'pranet':                  # lateral_map_2 lacks the background channel: prepend zeros
                    scores_raw0 = scores_raw[3]
                    scores_raw = torch.cat([torch.zeros_like(scores_raw0[:, [0]]), scores_raw0], dim=1)
                if model_type == 'nnunet':
                    scores_raw = scores_raw[0]
                scores_raw = scores_raw.float().contiguous()
                if scores_raw.dim() != 4 or scores_raw.shape[0] != B or scores_raw.shape[1] != K:
                    raise ValueError("test_single_batch: the net returned scores of shape %s, expected [%d, %d, h, w]"
                                     % (tuple(scores_raw.shape), B, K))
                h, w = scores_raw.shape[2:]
                L.call("sx_sw2d_accumulate", scores_raw.data_ptr(), B, K, h, w, dx, dy, preds.data_ptr(), cnt.data_ptr(),
                       H2, W2, xs, ys, m, wts, st())
                del test_patch, scores_raw                  # one variant's window alive at a time

    preds_soft = torch.empty((B, K, H, W), device=dev, dtype=torch.float32)
    preds_hard = torch.empty((B, K, H, W), device=dev, dtype=torch.int32)
    L.call("sx_sw2d_finalize", preds.data_ptr(), cnt.data_ptr(), B, K, H2, W2, hl_pad, wl_pad, H, W, preds_soft.data_ptr(),
           preds_hard.data_ptr(), st())
    return preds_hard, preds_soft
