"""Restatement of the 3-D batch preparation (checker only): the reference's brats_map_label and RandomResizedCrop
(code/dataloaders/datasets3d.py:16-40, :611-657) in stock PyTorch, with the crop's draws given as a record
(s_h, s_w, s_d, h_start, w_start, d_start) instead of drawn with torch.rand / torch.randint.

Both compute in the input's dtype on the input's device.  resized_crop resizes with F.interpolate, as the reference
does (tools/time_prep3d.py times its float32 form as the eager formulation).  In float64, F.interpolate would also
place its taps in float64, while the reference's float32 call places them in float32, which moves a tap by up to
~1e-6 cells; `resize=trilinear_f32_taps` restates the resize with the float32 tap positions and weights of PyTorch's
float32 kernels and blends in the input's dtype, which is what the tests compare with the fixtures in float64.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def brats_map_label(mask: torch.Tensor, binarize, dtype=torch.float32) -> torch.Tensor:
    """datasets3d.py:16-40 on the input's device; [B,...] inputs give the reference's permuted [B,K,...] view."""
    K = 2 if binarize else 4
    nhot = torch.zeros((K,) + tuple(mask.shape), device=mask.device, dtype=dtype)
    nhot[0, mask == 0] = 1
    if binarize:
        nhot[1, mask > 0] = 1
    else:
        nhot[1, mask == 3] = 1
        nhot[2, (mask == 3) | (mask == 1) | (mask == 2)] = 1
        nhot[3, (mask == 3) | (mask == 1)] = 1
    if nhot.dim() == 5:
        nhot = nhot.permute(1, 0, 2, 3, 4)
    return nhot


def crop_geometry(in_size, out_size, rec):
    """-> (resized sizes, F.pad's pads, starts) of a record, as the reference computes them: int(L * s) with s float32."""
    rec = torch.as_tensor(rec, dtype=torch.float32).reshape(6).cpu()
    resized = tuple(int(L * rec[a:a + 1]) for a, L in enumerate(in_size))
    pads = []
    for R, O in zip(resized, out_size):
        p = max(O - R, 0)
        pads.append((p // 2, p - p // 2))
    starts = tuple(int(v) for v in rec[3:])
    return resized, pads, starts


def _interpolate(x, size):
    return F.interpolate(x, size=size, mode="trilinear", align_corners=False)


def _taps_f32(L, R, device):
    """PyTorch's linear taps of an axis of L cells resized to R (align_corners=False) in float32:
    source = max((j + 0.5) * (L / R) - 0.5, 0), i0 = min(floor(source), L - 1), i1 = i0 + (i0 < L - 1), w1 = source - i0."""
    ratio = torch.tensor(L, dtype=torch.float32) / torch.tensor(R, dtype=torch.float32)
    src = ((torch.arange(R, dtype=torch.float32) + 0.5) * ratio - 0.5).clamp_min(0)
    i0 = src.long().clamp_max(L - 1)
    i1 = i0 + (i0 < L - 1).long()
    w1 = src - i0.float()
    return i0.to(device), i1.to(device), w1.to(device)


def trilinear_f32_taps(x, size):
    """F.interpolate(x, size, mode='trilinear', align_corners=False) with float32 taps, blended in x's dtype in PyTorch's
    order: along D first, then W, then H (upsample_trilinear3d's nesting)."""
    for dim, R in ((4, size[2]), (3, size[1]), (2, size[0])):
        i0, i1, w1 = _taps_f32(x.shape[dim], R, x.device)
        shape = [1] * 5
        shape[dim] = R
        w1 = w1.to(x.dtype).view(shape)
        x = (1 - w1) * x.index_select(dim, i0) + w1 * x.index_select(dim, i1)
    return x


def resized_crop(volume: torch.Tensor, mask: torch.Tensor, out_size, rec, resize=_interpolate):
    """datasets3d.py:626-665 with the record's draws: trilinear resize, zero padding, crop, in the inputs' dtype."""
    resized, pads, starts = crop_geometry(volume.shape[2:], out_size, rec)
    outs = []
    for x in (volume, mask):
        y = resize(x, resized)
        if any(p != (0, 0) for p in pads):
            y = F.pad(y, (pads[2][0], pads[2][1], pads[1][0], pads[1][1], pads[0][0], pads[0][1]), "constant", 0)
        (h, w, d), (H, W, D) = starts, out_size
        outs.append(y[:, :, h:h + H, w:w + W, d:d + D].clone())
    return tuple(outs)
