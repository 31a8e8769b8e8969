"""Plain-PyTorch restatement of the reference's 2-D evaluation (TEST INFRASTRUCTURE ONLY — see segtran_oracle.py header).

Follows code/test_util2d.py:151-265 (test_single_batch, calc_dice, calc_batch_metric), code/dataloaders/datasets2d.py:
178-196 (harden_segmap2d) and the unbatched branch of code/utils/losses.py:76-127 (calc_vcdr).  Device-agnostic: the
tensors' device is used throughout (the reference's ``device='cuda'`` accumulator follows the image here), so the same
code is the CPU checker and the on-GPU formulation tools/time_eval2d.py times.  Pinned by tests/golden/eval2d.pt, which
oracle/gen_eval2d_golden.py produces with the reference's own functions."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F


def harden_segmap2d(mask_soft, T=0.5):                                          # datasets2d.py:178-196
    mask_hard = (mask_soft >= T).int()
    if mask_hard.dim() == 4:
        mask_hard[:, 0] = (mask_hard[:, 1:].sum(dim=1) == 0)
    else:
        mask_hard[0] = (mask_hard[1:].sum(dim=0) == 0)
    return mask_hard


def test_single_batch(net, image_batch, orig_input_size, patch_size, stride, task_name, num_classes, model_type):
    B, C, H, W = image_batch.shape
    dx, dy = orig_input_size
    h_pad, w_pad = max(dx - H, 0), max(dy - W, 0)                               # :153-166
    add_pad = (h_pad + w_pad) > 0
    hl_pad, wl_pad = h_pad // 2, w_pad // 2
    if add_pad:
        image_batch = F.pad(image_batch, (wl_pad, w_pad - wl_pad, hl_pad, h_pad - hl_pad), mode='constant', value=0)
    H2, W2 = image_batch.shape[2:]
    sx = math.ceil((H2 - dx) / stride[0]) + 1                                   # :173-174
    sy = math.ceil((W2 - dy) / stride[1]) + 1
    preds_soft = torch.zeros((B, num_classes, H2, W2), device=image_batch.device)
    cnt = torch.zeros_like(preds_soft[:, 0])
    for x in range(sx):                                                         # :181-214
        xs = min(stride[0] * x, H2 - dx)
        for y in range(sy):
            ys = min(stride[1] * y, W2 - dy)
            patch = F.interpolate(image_batch[:, :, xs:xs + dx, ys:ys + dy], size=patch_size, mode='bilinear',
                                  align_corners=False)
            with torch.no_grad():
                scores = net(patch)
            if model_type == 'pranet':
                s0 = scores[3]
                scores = torch.cat([torch.zeros_like(s0[:, [0]]), s0], dim=1)
            if model_type == 'nnunet':
                scores = scores[0]
            scores = F.interpolate(scores, size=orig_input_size, mode='bilinear', align_corners=False)
            preds_soft[:, :, xs:xs + dx, ys:ys + dy] += torch.sigmoid(scores)
            cnt[:, xs:xs + dx, ys:ys + dy] += 1
    preds_soft = preds_soft / cnt.unsqueeze(dim=1)                              # :216-217
    preds_hard = harden_segmap2d(preds_soft)
    if add_pad:                                                                 # :219-221
        preds_hard = preds_hard[:, :, hl_pad:hl_pad + H, wl_pad:wl_pad + W]
        preds_soft = preds_soft[:, :, hl_pad:hl_pad + H, wl_pad:wl_pad + W]
    return preds_hard, preds_soft


def calc_dice(predictions, gt_mask):                                            # test_util2d.py:229-236
    gt_mask = gt_mask.float()
    smooth = 1e-5
    intersect = torch.sum(predictions * gt_mask, dim=(-1, -2))
    y_sum = torch.sum(gt_mask * gt_mask, dim=(-1, -2))
    z_sum = torch.sum(predictions * predictions, dim=(-1, -2))
    return (2 * intersect + smooth) / (z_sum + y_sum + smooth)


def calc_vcdr(mask_nhot_soft, thres=0.5, delta=1):                               # losses.py:102-127 (no batch dim)
    mask_nhot = mask_nhot_soft >= thres
    vert_indices = torch.arange(1, mask_nhot.shape[1] + 1, 1, device=mask_nhot_soft.device)
    disc_vert_indices = vert_indices[mask_nhot[1].sum(dim=1) > 0]
    if len(disc_vert_indices) == 0:
        return torch.tensor(-1., device=mask_nhot.device)
    disc_vert_len = disc_vert_indices.max() - disc_vert_indices.min() - delta
    cup_vert_indices = vert_indices[mask_nhot[2].sum(dim=1) > 0]
    if len(cup_vert_indices) == 0:
        return torch.tensor(0., device=mask_nhot.device)
    cup_vert_len = cup_vert_indices.max() - cup_vert_indices.min() - delta
    return cup_vert_len / (disc_vert_len + 0.0001)


def calc_batch_metric(BC_pred_soft, BC_gt, num_classes, do_calc_vcdr_error=False):   # test_util2d.py:241-265
    batch_size = len(BC_pred_soft)
    out = np.zeros((batch_size, num_classes - 1 + do_calc_vcdr_error))
    for ins in range(batch_size):
        C_gt = BC_gt[ins]
        C_pred_soft = F.interpolate(BC_pred_soft[ins].unsqueeze(0), size=C_gt.shape[1:], mode='bilinear',
                                    align_corners=False)[0]
        C_pred = harden_segmap2d(C_pred_soft)
        for cls in range(1, num_classes):
            out[ins, cls - 1] = calc_dice(C_pred[cls], C_gt[cls]).cpu().numpy()
        if do_calc_vcdr_error:
            out[ins, num_classes - 1] = np.abs((calc_vcdr(C_gt) - calc_vcdr(C_pred)).cpu().numpy())
    return out


def fundus_like_gt(B, H, W, seed, jitter=0.0, jitter_seed=0):
    """[B,3,H,W] float 0/1 ground truths shaped like REFUGE masks: an elliptical disc (class 1) containing an elliptical
    cup (class 2), class 0 their complement, with per-image centres and radii drawn from `seed`.  jitter > 0 scales each
    radius by a factor in [1 - jitter/2, 1 + jitter/2] drawn from `jitter_seed` (a prediction-like variant)."""
    g = torch.Generator().manual_seed(seed)
    gj = torch.Generator().manual_seed(jitter_seed)
    yy = torch.arange(H, dtype=torch.float64).view(H, 1)
    xx = torch.arange(W, dtype=torch.float64).view(1, W)
    out = torch.zeros(B, 3, H, W)
    for b in range(B):
        u = torch.rand(6, generator=g, dtype=torch.float64)
        f = 1 + jitter * (torch.rand(4, generator=gj, dtype=torch.float64) - 0.5)
        cy, cx = H * (0.4 + 0.2 * u[0]), W * (0.4 + 0.2 * u[1])
        ry, rx = H * (0.18 + 0.1 * u[2]), W * (0.15 + 0.1 * u[3])
        d = ((yy - cy) / (ry * f[0])) ** 2 + ((xx - cx) / (rx * f[1])) ** 2 <= 1
        cry, crx = ry * f[2] * (0.35 + 0.25 * u[4]), rx * f[3] * (0.35 + 0.25 * u[5])
        c = ((yy - cy) / cry) ** 2 + ((xx - cx) / crx) ** 2 <= 1
        out[b, 1] = d.float()
        out[b, 2] = c.float()
        out[b, 0] = 1 - torch.clamp(out[b, 1] + out[b, 2], max=1)
    return out


def soft_from_gt(gt, h, w, seed, noise=0.35):
    """A soft prediction [B,K,h,w] from a 0/1 map: resized to h x w, pulled towards 0.5 and perturbed by uniform noise,
    so the hardened masks differ from the map along the borders."""
    g = torch.Generator().manual_seed(seed)
    s = F.interpolate(gt.float(), size=(h, w), mode='bilinear', align_corners=False)
    return (0.15 + 0.7 * s + noise * (torch.rand(s.shape, generator=g) - 0.5)).clamp(0, 1)
