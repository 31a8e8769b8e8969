"""GPU drop-ins for the batch preparation of the reference's 3-D training loop (code/train3d.py:711-715), with the
names and signatures of code/dataloaders/datasets3d.py:

  brats_map_label(mask, binarize)                               datasets3d.py:16-40   (also test_util3d.py:38)
  RandomResizedCrop(volume, mask, out_size, crop_percents, ...) datasets3d.py:611-657 (--randscale)
  draw_resized_crop(in_size, out_size, crop_percents, ...)      the draws of RandomResizedCrop, on the device

Each function is one pass over the data in one kernel of csrc/sx_prep3d.cu.  The resized crop gathers the trilinear taps
of every output voxel straight from its input, so the resized and padded intermediate is never allocated.  The crop's
scale and starts are drawn by a one-thread kernel from a device seed (ops.new_dropout_seed), so nothing here
synchronises with the host and a captured training step draws a new crop on every replay after ops.advance_seed.  The
one deviation from the reference: the draws follow the reference's distributions but come from the library's device
generator, so torch.manual_seed does not select them; given the same draws, the result is the reference's.
No autograd (the inputs are data) and no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib as L
from . import ops

_LABEL_TYPES = {torch.uint8: L.SX_LABEL_U8, torch.int16: L.SX_LABEL_I16, torch.int32: L.SX_LABEL_I32,
                torch.int64: L.SX_LABEL_I64, torch.float32: L.SX_LABEL_F32}


def brats_map_label(mask: torch.Tensor, binarize) -> torch.Tensor:
    """Drop-in for datasets3d.brats_map_label on a CUDA label tensor [B,H,W,D] or [H,W,D] (uint8, int16, int32, int64 or
    float32).  -> contiguous fp32 [B,K,H,W,D] / [K,H,W,D] on the label's device, K = 2 if binarize else 4: class 0 is
    label == 0; binarized, class 1 is label > 0; otherwise ET (3), WT (1, 2, 3) and TC (1, 3).  Other values (4, 255,
    negative ones) fall in no class of the 4-class map; positive ones are foreground in the binarized map, as in the
    reference.  The reference returns the batched map as a permuted view; this one has the same values, contiguous."""
    if not isinstance(mask, torch.Tensor):
        raise ValueError("brats_map_label: a label tensor expected, got %s" % type(mask).__name__)
    if mask.dim() not in (3, 4):
        raise ValueError("brats_map_label: labels [B,H,W,D] or [H,W,D] expected, got %s" % (tuple(mask.shape),))
    if mask.dtype not in _LABEL_TYPES:
        raise ValueError("brats_map_label: label dtype %s not supported (uint8, int16, int32, int64, float32)"
                         % mask.dtype)
    ops._req_cuda(mask)
    K = 2 if binarize else 4
    lab = mask.contiguous()
    batched = lab.dim() == 4
    B = lab.shape[0] if batched else 1
    V = lab[0].numel() if batched else lab.numel()
    out = torch.empty(((B,) if batched else ()) + (K,) + tuple(lab.shape[-3:]), device=lab.device, dtype=torch.float32)
    if out.numel():
        L.call("sx_brats_map_label", lab.data_ptr(), _LABEL_TYPES[lab.dtype], B, V, 1 if binarize else 0,
               out.data_ptr(), ops._stream())
    return out


def _sizes(size, what):
    s = tuple(int(v) for v in size)
    if len(s) != 3 or min(s) < 1:
        raise ValueError("%s: three positive sizes (H, W, D) expected, got %r" % (what, size))
    return s


def _scale_range(in_size, crop_percents, what):
    min_crop, max_crop = crop_percents
    min_scale, max_scale = 1 + min_crop, 1 + max_crop
    if min_scale <= 0:
        raise ValueError("%s: 1 + min_crop must be positive, got crop_percents %r" % (what, tuple(crop_percents)))
    if max_scale < min_scale:
        raise ValueError("%s: crop_percents %r has max < min" % (what, tuple(crop_percents)))
    smin = float(torch.tensor(min_scale, dtype=torch.float32))
    for Lh in in_size:
        # the reference's int(L * s) in float32; an empty intermediate axis is an error there (F.interpolate)
        if int(torch.tensor(float(Lh), dtype=torch.float32) * smin) < 1:
            raise ValueError("%s: a scale of %g leaves an axis of %d cells empty" % (what, min_scale, Lh))
    return min_scale, max_scale


def _draw(in_size, out_size, scale_range, isotropic, seed, device) -> torch.Tensor:
    min_scale, max_scale = scale_range
    if seed is None:
        seed = ops.new_dropout_seed(device)
    elif isinstance(seed, torch.Tensor):
        ops._req_cuda(seed)
        if seed.dtype != torch.int64 or seed.numel() != 1:
            raise ValueError("draw_resized_crop: seed must be an int or a one-element int64 device tensor")
    sv, sp = ops._seed_args(seed)
    rec = torch.empty(6, device=device, dtype=torch.float32)
    L.call("sx_draw_resized_crop", sp, sv, *in_size, *out_size, float(min_scale), float(max_scale),
           1 if isotropic else 0, rec.data_ptr(), ops._stream())
    return rec


def draw_resized_crop(in_size, out_size, crop_percents, isotropic=True, seed=None) -> torch.Tensor:
    """The draws of RandomResizedCrop as a float32 device record (s_h, s_w, s_d, h_start, w_start, d_start):
    s ~ U[1+min_crop, 1+max_crop) (one draw for all axes when isotropic, else three in H, W, D order), then each start
    uniform on [0, padded_len - out_len] with padded_len = max(int(L * s), out_len).  One tiny kernel, no host
    synchronisation.  seed: None draws a per-call seed from the device generator (ops.new_dropout_seed: a captured step
    that calls ops.advance_seed draws anew on each replay); an int or an int64 device tensor fixes it.  The record is on
    the seed tensor's device, else on the current CUDA device."""
    in_size, out_size = _sizes(in_size, "draw_resized_crop"), _sizes(out_size, "draw_resized_crop")
    scale_range = _scale_range(in_size, crop_percents, "draw_resized_crop")
    if isinstance(seed, torch.Tensor):
        device = seed.device
    else:
        device = torch.device("cuda", torch.cuda.current_device())
    return _draw(in_size, out_size, scale_range, isotropic, seed, device)


def _operand(t: torch.Tensor, out: torch.Tensor) -> L.sx_crop_operand:
    op = L.sx_crop_operand()
    op.x = t.data_ptr()
    for i, s in enumerate(t.stride()):
        op.stride[i] = s
    op.y = out.data_ptr()
    op.C = t.shape[1]
    return op


def RandomResizedCrop(volume: torch.Tensor, mask: torch.Tensor, out_size, crop_percents, isotropic=True, *, draws=None,
                      seed=None):
    """Drop-in for datasets3d.RandomResizedCrop on CUDA fp32 tensors volume [B,Cv,H,W,D] and mask [B,Cm,H,W,D] (any
    strides: the reference's permuted n-hot view works as is).  -> (volume3, mask3), contiguous [B,C,*out_size]: both
    resized trilinearly (align_corners=False) to (int(H s_h), int(W s_w), int(D s_d)), zero-padded to at least out_size
    (pad // 2 before, the rest after) and cropped at the record's starts; the whole batch shares one scale and one crop.
    One kernel: each output voxel gathers its <= 8 taps per channel from the inputs, 0 in the padding.
    draws: None draws the record on the device (draw_resized_crop; `seed` as there); otherwise a float32 record
    (s_h, s_w, s_d, h_start, w_start, d_start) on the host or the device, used as given.  Cells of a record's crop that
    lie outside the padded intermediate are 0."""
    if not isinstance(volume, torch.Tensor) or not isinstance(mask, torch.Tensor):
        raise ValueError("RandomResizedCrop: volume and mask must be tensors")
    if volume.dim() != 5 or mask.dim() != 5:
        raise ValueError("RandomResizedCrop: 5-D volume and mask [B,C,H,W,D] expected, got %s and %s"
                         % (tuple(volume.shape), tuple(mask.shape)))
    if volume.shape[0] != mask.shape[0] or volume.shape[2:] != mask.shape[2:]:
        raise ValueError("RandomResizedCrop: volume %s and mask %s differ in batch or spatial size"
                         % (tuple(volume.shape), tuple(mask.shape)))
    in_size = tuple(int(v) for v in volume.shape[2:])
    out_size = _sizes(out_size, "RandomResizedCrop")
    scale_range = _scale_range(in_size, crop_percents, "RandomResizedCrop")
    rec = None
    if draws is not None:
        rec = torch.as_tensor(draws, dtype=torch.float32)
        if rec.numel() != 6:
            raise ValueError("RandomResizedCrop: draws must hold 6 values (s_h, s_w, s_d, h_start, w_start, d_start)")
    ops._req_cuda(volume, mask)
    if volume.dtype != torch.float32 or mask.dtype != torch.float32:
        raise ValueError("RandomResizedCrop: fp32 volume and mask expected, got %s and %s" % (volume.dtype, mask.dtype))
    if volume.device != mask.device:
        raise ValueError("RandomResizedCrop: volume on %s, mask on %s" % (volume.device, mask.device))
    dev = volume.device
    if rec is None:
        rec = _draw(in_size, out_size, scale_range, isotropic, seed, dev)
    else:
        rec = rec.reshape(6).to(dev).contiguous()
    B = volume.shape[0]
    vout = torch.empty((B, volume.shape[1]) + out_size, device=dev, dtype=torch.float32)
    mout = torch.empty((B, mask.shape[1]) + out_size, device=dev, dtype=torch.float32)
    pairs = [(t, o) for t, o in ((volume, vout), (mask, mout)) if t.shape[1] > 0]
    if B > 0 and pairs:
        a = _operand(*pairs[0])
        b = _operand(*pairs[1]) if len(pairs) > 1 else None
        L.call("sx_resized_crop", C.byref(a), None if b is None else C.byref(b), B, *in_size, *out_size,
               rec.data_ptr(), ops._stream())
    return vout, mout
