"""Stock-PyTorch restatement of mirror test-time augmentation (``mirror_axes`` of segtran_b200.inference, beyond the
reference) (TEST INFRASTRUCTURE ONLY — see segtran_oracle.py header).

The sliding windows, padding and post-process follow oracle/infer_oracle.py (3-D) and oracle/eval2d_oracle.py (2-D);
each window batch x is also predicted as flip_m(net(flip_m(x))) with torch.flip for every variant m.  Device-agnostic:
the same code is the CPU checker of tests/golden/tta_*.pt (oracle/gen_tta_golden.py) and the torch.flip formulation the
GPU tests compare against."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.eval2d_oracle import harden_segmap2d
from oracle.infer_oracle import make_brats_pred_consistent
def mirror_dims(mirror_axes, lead):
    """The dims torch.flip reverses for each of the 2^k variants (bit i mirrors mirror_axes[i]), spatial axes offset by
    the `lead` batch and channel dims."""
    return [[lead + a for i, a in enumerate(mirror_axes) if m >> i & 1] for m in range(1 << len(mirror_axes))]


def _flip(x, dims):
    return torch.flip(x, dims) if dims else x


def test_single_case_tta(net, image, orig_patch_size, input_patch_size, batch_size, stride_xy, stride_z, task_name, net_type,
                         num_classes, mirror_axes):
    """test_single_case with each window batch x also predicted as flip_m(net(flip_m(x))) for every variant m, all
    variants pooled into one average before the BraTS rule / arg-max."""
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
                            preds_soft[:, xs:xs + dx, ys_i:ys_i + dy, zs_i:zs_i + dz] += probs[i]
                            cnt[xs:xs + dx, ys_i:ys_i + dy, zs_i:zs_i + dz] += 1
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


def test_single_batch_tta(net, image_batch, orig_input_size, patch_size, stride, task_name, num_classes, model_type,
                          mirror_axes):
    """test_util2d.test_single_batch with each window x also predicted as flip_m(net(flip_m(x))) for every variant m,
    all variants pooled into one average before harden_segmap2d."""
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
                preds_soft[:, :, xs:xs + dx, ys:ys + dy] += torch.sigmoid(scores)
                cnt[:, xs:xs + dx, ys:ys + dy] += 1
    preds_soft = preds_soft / cnt.unsqueeze(dim=1)
    preds_hard = harden_segmap2d(preds_soft)
    if add_pad:
        preds_hard = preds_hard[:, :, hl_pad:hl_pad + H, wl_pad:wl_pad + W]
        preds_soft = preds_soft[:, :, hl_pad:hl_pad + H, wl_pad:wl_pad + W]
    return preds_hard, preds_soft


class AsymNet(torch.nn.Module):
    """Stand-in net of the TTA fixtures that is deliberately NOT mirror-equivariant, yet element-wise reproducible on any
    device: class k's score = a[k]·x[:,ch[k]] + b[k] + g[k]·(x[:,ch[k]] rolled by one cell along every spatial axis)
    + r[k]·Σ_axis index/size."""

    def __init__(self, a, b, ch, g, r):
        super().__init__()
        self.a, self.b, self.g, self.r = ([float(v) for v in t] for t in (a, b, g, r))
        self.ch = [int(c) for c in ch]

    @staticmethod
    def params(K, C, seed):
        gen = torch.Generator().manual_seed(seed)
        u = lambda lo, hi: [float(v) for v in lo + (hi - lo) * torch.rand(K, generator=gen)]     # noqa: E731
        return dict(a=u(0.8, 1.6), b=u(-0.5, 0.5), ch=[k % C for k in range(K)], g=u(0.3, 0.9), r=u(-2.0, 2.0))

    def forward(self, x):
        sp = tuple(range(2, x.dim()))
        ramp = 0.
        for d in sp:
            n = x.shape[d]
            shape = [1] * (x.dim() - 1)
            shape[d - 1] = n
            ramp = ramp + (torch.arange(n, device=x.device, dtype=torch.float32) / n).view(shape[1:])
        outs = []
        for a, b, g, r, c in zip(self.a, self.b, self.g, self.r, self.ch):
            xc = x[:, c]
            outs.append(((xc * a + b) + torch.roll(xc, (1,) * len(sp), tuple(d - 1 for d in sp)) * g) + ramp * r)
        return torch.stack(outs, dim=1)
