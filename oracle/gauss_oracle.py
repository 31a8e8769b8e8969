"""Stock-PyTorch restatement of Gaussian window blending (``gaussian_sigma_scale`` of segtran_b200.inference, beyond the
reference) (TEST INFRASTRUCTURE ONLY — see segtran_oracle.py header).

The sliding windows, padding, mirror variants and post-process follow oracle/infer_oracle.py and oracle/tta_oracle.py
(3-D) and oracle/eval2d_oracle.py (2-D); the only change is the update: every window (and every mirror variant of it)
adds ``weight * sigmoid(scores)`` to the soft map and ``weight`` to the count, with ``weight`` a map of the window's
shape.  ``gaussian_weight`` restates the weight formula on its own, independently of the product package.  With a map
of ones the functions are the plain / TTA oracles, which pins them to the reference-generated fixtures.  Device-agnostic:
the same code is the CPU checker and the formulation the GPU tests compare against."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.eval2d_oracle import harden_segmap2d
from oracle.infer_oracle import make_brats_pred_consistent
from oracle.tta_oracle import mirror_dims

MIN_WEIGHT = 1e-3          # MONAI's floor of the importance map


def gaussian_axis(d, sigma_scale):
    """fp32 [d]: exp(-(i - (d-1)/2)^2 / (2 (s d)^2)) in float64, divided by its maximum over i, then rounded."""
    i = torch.arange(d, dtype=torch.float64)
    sigma = torch.tensor(sigma_scale * d, dtype=torch.float64)
    g = torch.exp(-(i - (d - 1) / 2) ** 2 / (2 * sigma ** 2))
    return (g / g.max()).float()


def gaussian_weight(size, sigma_scale):
    """fp32 map of the window shape ``size`` (2 or 3 axes): max(g_0(i) * g_1(j) [* g_2(l)], 1e-3), the product in fp32
    in axis order."""
    w = None
    for a, d in enumerate(size):
        shape = [1] * len(size)
        shape[a] = d
        g = gaussian_axis(d, sigma_scale).view(shape)
        w = g if w is None else w * g
    return w.clamp_min(MIN_WEIGHT)


def _flip(x, dims):
    return torch.flip(x, dims) if dims else x


def test_single_case_gauss(net, image, orig_patch_size, input_patch_size, batch_size, stride_xy, stride_z, task_name,
                           net_type, num_classes, mirror_axes, weight):
    """test_single_case (with mirror_axes as in tta_oracle) where each window adds weight * probs and weight;
    weight: [dx, dy, dz] fp32."""
    C, H, W, D = image.shape
    dx, dy, dz = orig_patch_size
    h_pad, w_pad, d_pad = max(dx - H, 0), max(dy - W, 0), max(dz - D, 0)
    add_pad = (h_pad + w_pad + d_pad) > 0
    hl, wl, dl = h_pad // 2, w_pad // 2, d_pad // 2
    if add_pad:
        image = F.pad(image, (dl, d_pad - dl, wl, w_pad - wl, hl, h_pad - hl), mode='constant', value=0)
    C, H2, W2, D2 = image.shape
    sx = math.ceil((H2 - dx) / stride_xy) + 1
    sy = math.ceil((W2 - dy) / stride_xy) + 1
    sz = math.ceil((D2 - dz) / stride_z) + 1
    preds_soft = torch.zeros((num_classes,) + tuple(image.shape[1:]), device=image.device)
    cnt = torch.zeros_like(image[0], dtype=torch.float32)
    weight = weight.to(image.device)
    variants = mirror_dims(mirror_axes, 2)
    for x in range(sx):
        xs = min(stride_xy * x, H2 - dx)
        yzs, patches = [], []
        for y in range(sy):
            ys = min(stride_xy * y, W2 - dy)
            for z in range(sz):
                zs = min(stride_z * z, D2 - dz)
                patches.append(image[:, xs:xs + dx, ys:ys + dy, zs:zs + dz])
                yzs.append((ys, zs))
                if len(patches) == batch_size or (y == sy - 1 and z == sz - 1):
                    batch = F.interpolate(torch.stack(patches, 0), size=input_patch_size, mode='trilinear', align_corners=False)
                    for dims in variants:
                        with torch.no_grad():
                            scores = net(_flip(batch, dims))
                        if net_type == 'unet':
                            scores = scores[1]
                        scores = F.interpolate(_flip(scores, dims), size=orig_patch_size, mode='trilinear',
                                               align_corners=False)
                        probs = torch.sigmoid(scores)
                        for i, (ys_i, zs_i) in enumerate(yzs):
                            preds_soft[:, xs:xs + dx, ys_i:ys_i + dy, zs_i:zs_i + dz] += weight * probs[i]
                            cnt[xs:xs + dx, ys_i:ys_i + dy, zs_i:zs_i + dz] += weight
                    patches, yzs = [], []
    preds_soft = preds_soft / cnt.unsqueeze(0)
    if task_name == 'brats':
        preds_soft = make_brats_pred_consistent(preds_soft)
        preds_hard = torch.zeros_like(preds_soft)
        preds_hard[1:] = (preds_soft[1:] >= 0.5)
        preds_hard[0] = (preds_hard[1:].sum(dim=0) == 0)
    else:
        preds_hard = torch.argmax(preds_soft, dim=0)
    if add_pad:
        preds_hard = preds_hard[..., hl:hl + H, wl:wl + W, dl:dl + D].clone()
        preds_soft = preds_soft[:, hl:hl + H, wl:wl + W, dl:dl + D].clone()
    return preds_hard, preds_soft


def test_single_batch_gauss(net, image_batch, orig_input_size, patch_size, stride, task_name, num_classes, model_type,
                            mirror_axes, weight):
    """test_util2d.test_single_batch (with mirror_axes as in tta_oracle) where each window adds weight * probs and
    weight, on the upsampled window; weight: [dx, dy] fp32."""
    B, C, H, W = image_batch.shape
    dx, dy = orig_input_size
    h_pad, w_pad = max(dx - H, 0), max(dy - W, 0)
    add_pad = (h_pad + w_pad) > 0
    hl_pad, wl_pad = h_pad // 2, w_pad // 2
    if add_pad:
        image_batch = F.pad(image_batch, (wl_pad, w_pad - wl_pad, hl_pad, h_pad - hl_pad), mode='constant', value=0)
    H2, W2 = image_batch.shape[2:]
    sx = math.ceil((H2 - dx) / stride[0]) + 1
    sy = math.ceil((W2 - dy) / stride[1]) + 1
    preds_soft = torch.zeros((B, num_classes, H2, W2), device=image_batch.device)
    cnt = torch.zeros_like(preds_soft[:, 0])
    weight = weight.to(image_batch.device)
    variants = mirror_dims(mirror_axes, 2)
    for x in range(sx):
        xs = min(stride[0] * x, H2 - dx)
        for y in range(sy):
            ys = min(stride[1] * y, W2 - dy)
            patch = F.interpolate(image_batch[:, :, xs:xs + dx, ys:ys + dy], size=patch_size, mode='bilinear',
                                  align_corners=False)
            for dims in variants:
                with torch.no_grad():
                    scores = net(_flip(patch, dims))
                if model_type == 'pranet':
                    s0 = scores[3]
                    scores = torch.cat([torch.zeros_like(s0[:, [0]]), s0], dim=1)
                if model_type == 'nnunet':
                    scores = scores[0]
                scores = F.interpolate(_flip(scores, dims), size=orig_input_size, mode='bilinear', align_corners=False)
                preds_soft[:, :, xs:xs + dx, ys:ys + dy] += weight * torch.sigmoid(scores)
                cnt[:, xs:xs + dx, ys:ys + dy] += weight
    preds_soft = preds_soft / cnt.unsqueeze(dim=1)
    preds_hard = harden_segmap2d(preds_soft)
    if add_pad:
        preds_hard = preds_hard[:, :, hl_pad:hl_pad + H, wl_pad:wl_pad + W]
        preds_soft = preds_soft[:, :, hl_pad:hl_pad + H, wl_pad:wl_pad + W]
    return preds_hard, preds_soft
