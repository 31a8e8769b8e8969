"""Training-step tail of the hot path (SURVEY.md §8 f.2): the reference's segmentation loss and its BertAdam update,
as device-resident kernels behind the same call shapes the reference training loop uses.

  seg_loss(logits, mask, pos_weight, class_weights, dice_w)   train3d.py:731-756 + utils/losses.py:47-60
  attn_consist_loss3d / attn_consist_loss2d                    train3d.py:426-449 / train2d.py:668-723 (--attnconsist)
  FlatBertAdam(param_groups, ..., bucket=GradBucket)           optimization.py:43-164 + train3d.py:760-761 (--gradclip)

Nothing here synchronises with the host: the loss, the clip coefficients, the scheduled learning rates and the step
counter live on the GPU, so forward + loss + backward + update can sit in one CUDA graph.  No CPU fallback.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import _lib as L
from . import ops


# ------------------------------------------------------------------------------------------------------------------
# loss
# ------------------------------------------------------------------------------------------------------------------
class _SegLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, mask, pos_weight, class_w, dice_w):
        ops._req_cuda(logits, mask, pos_weight, class_w)
        if logits.dtype != torch.float32 or mask.dtype != torch.float32 or logits.shape != mask.shape:
            raise L.SxError("seg_loss: fp32 logits and an n-hot fp32 mask of the same [B,K,*spatial] shape expected")
        logits, mask = logits.contiguous(), mask.contiguous()
        B, K = logits.shape[:2]
        V = logits[0, 0].numel()
        dev = logits.device
        pw = None if pos_weight is None else pos_weight.to(dev, torch.float32).contiguous()
        cw = None if class_w is None else class_w.to(dev, torch.float32).contiguous()
        sums = torch.empty(B * K * 4, device=dev, dtype=torch.float64)
        out3 = torch.empty(3, device=dev, dtype=torch.float32)
        coef = torch.empty(B * K * 2, device=dev, dtype=torch.float32)
        L.call("sx_seg_loss_fwd", logits.data_ptr(), mask.data_ptr(), B, K, V, ops._ptr(pw), ops._ptr(cw), float(dice_w),
               sums.data_ptr(), out3.data_ptr(), coef.data_ptr(), ops._stream())
        ctx.save_for_backward(logits, mask, pw, coef)
        ctx.meta = (B, K, V, float(dice_w))
        return out3                                  # {loss, ce, dice}; only element 0 is differentiated

    @staticmethod
    def backward(ctx, g3):
        logits, mask, pw, coef = ctx.saved_tensors
        B, K, V, dice_w = ctx.meta
        d = torch.empty_like(logits)
        g = g3.contiguous().float()                  # g[0] = d(objective)/d(loss), read on the device
        L.call("sx_seg_loss_bwd", logits.data_ptr(), mask.data_ptr(), B, K, V, ops._ptr(pw), coef.data_ptr(),
               (1.0 - dice_w) / (float(B) * K * V), g.data_ptr(), d.data_ptr(), ops._stream())
        return d, None, None, None, None


def seg_loss(logits: torch.Tensor, mask: torch.Tensor, pos_weight: Optional[torch.Tensor] = None,
             class_weights: Optional[torch.Tensor] = None, dice_w: float = 0.5):
    """(loss, ce, dice) as 0-dim device tensors: loss = (1-dice_w) * BCEWithLogitsLoss(pos_weight)(logits, mask) +
    dice_w * sum_{k>=1} class_weights[k] * dice_loss_indiv(sigmoid(logits[:,k]), mask[:,k])   (train3d.py:738-756).
    One pass over the logits for the sums, one for the gradient; ce and dice are returned for logging."""
    o = _SegLoss.apply(logits, mask, pos_weight, class_weights, dice_w)
    return o[0], o[1].detach(), o[2].detach()


def _attn_consist_loss(layers_attn_scores, orig_feat_shape, mask, only_first_layer, variant):
    grid = tuple(int(s) for s in orig_feat_shape)
    if variant == ops.CONSIST_BCE:
        if mask.dim() != 5 or len(grid) != 3:
            raise ValueError("attn_consist_loss3d: mask [B,C,H,W,D] and a 3-D orig_feat_shape expected")
        mask = mask.permute(0, 1, 4, 2, 3)                 # (train3d.py:429) [B,C,D,H,W], resized to orig_feat_shape
    elif mask.dim() != 4 or len(grid) != 2:
        raise ValueError("attn_consist_loss2d: mask [B,C,H,W] and a 2-D orig_feat_shape expected")
    B, K = mask.shape[:2]
    N = 1
    for s in grid:
        N *= s
    n = 1 if only_first_layer else len(layers_attn_scores)
    entries = list(layers_attn_scores[:n])
    for e in entries:
        t = e[1] if isinstance(e, (list, tuple)) else e        # ator_out_scores [B,1,N,A] / dense [B,1,N,N]
        if t.shape[0] != B:
            raise ValueError("attn_consist_loss: the mask has batch %d, the attention scores %d" % (B, t.shape[0]))
        if t.shape[-2] != N or (not isinstance(e, (list, tuple)) and t.shape[-1] != N):
            raise ValueError("attn_consist_loss: %d tokens in the attention scores, orig_feat_shape %s has %d"
                             % (t.shape[-2], grid, N))
    if K > 16:
        raise ValueError("attn_consist_loss: %d mask channels (at most 16 supported)" % K)
    with torch.no_grad():                                  # linear resize, align_corners=False, one pass per axis
        F = ops.resize_linear(mask.to(torch.float32), grid).reshape(B, K, N).contiguous()
    cap = torch.zeros(2, device=F.device, dtype=torch.float32) if variant == ops.CONSIST_MARGIN else None
    total = None
    for e in entries:
        l = ops.attn_consist(e, F, variant, cap, 1.0 / n)
        total = l if total is None else ops.add(total, l)
    loss = ops.scale(total, 1.0 / n)
    if cap is not None:                                    # `if loss > 1: loss /= loss.item()`, factor kept on the device
        loss = ops.dot(loss, cap[1:2]).reshape(())
    return loss


def attn_consist_loss3d(layers_attn_scores, orig_feat_shape, mask, only_first_layer=True):
    """train3d.py:426-449 as a drop-in: mean BCE-with-logits of each layer's token affinity X (ator_out . in_ator for a
    squeezed layer, the [B,1,N,N] scores otherwise) against clip(F^T F, 0, 1) of the mask resized to orig_feat_shape,
    averaged over the first layer or all of them.  mask [B,C,H,W,D]; orig_feat_shape (D2,H2,W2)-ordered as the reference
    resizes it.  A 0-dim device tensor; X and the target matrix are never stored."""
    return _attn_consist_loss(layers_attn_scores, orig_feat_shape, mask, only_first_layer, ops.CONSIST_BCE)


def attn_consist_loss2d(layers_attn_scores, orig_feat_shape, mask, only_first_layer=False):
    """train2d.py:668-723 as a drop-in: per layer, the mean |x - mu_b| over the pairs whose affinity sits on the wrong side
    of the batch mean mu_b (same-class pairs below it, other pairs above mu_b - 0.1); averaged over the layers and capped
    at 1 (the reference's `loss /= loss.item()` becomes a device-side factor).  mask [B,C,H,W]."""
    return _attn_consist_loss(layers_attn_scores, orig_feat_shape, mask, only_first_layer, ops.CONSIST_MARGIN)


# ------------------------------------------------------------------------------------------------------------------
# optimiser
# ------------------------------------------------------------------------------------------------------------------
_SEG = 4096          # elements of one parameter handled by one thread block


class FlatBertAdam:
    """The reference's BertAdam (optimization.py:43-164: per-parameter gradient-norm clip `max_grad_norm`, Adam moments
    without bias correction, decoupled weight decay, warm-up schedule) plus the training loop's global clip
    (`--gradclip`, train3d.py:760-761), as ONE pass over flat buckets.

    `param_groups` is what the reference hands to BertAdam (train3d.py:334-339): dicts with 'params', 'lr' and
    'weight_decay'; a plain parameter iterable with the `lr=` / `weight_decay=` keywords also works.  The parameters
    are re-pointed into one contiguous fp32 buffer (their values are preserved), the gradients are the views of
    `bucket` (a parallel.GradBucket over the same parameters, created here when not given).  Differences from the
    reference, by design: gradients are not modified in place by the clips, and a parameter is skipped when its
    gradient is exactly zero (the reference skips `p.grad is None`)."""

    def __init__(self, param_groups, lr: float = None, warmup: float = -1, t_total: int = -1,
                 schedule: str = "warmup_linear", b1: float = 0.9, b2: float = 0.999, e: float = 1e-6,
                 weight_decay: float = 0.05, max_grad_norm: float = 0.05, grad_clip: float = -1.0, bucket=None):
        groups = list(param_groups)
        if groups and not isinstance(groups[0], dict):
            groups = [{"params": groups}]
        if schedule not in ("warmup_linear", "warmup_constant"):
            raise ValueError("FlatBertAdam: schedule %r not implemented (warmup_linear | warmup_constant)" % schedule)
        per = {}
        for gr in groups:
            glr = gr.get("lr", lr)
            if glr is None:
                raise ValueError("FlatBertAdam: no learning rate for a parameter group")
            for p in gr["params"]:
                if p.requires_grad and id(p) not in per:
                    per[id(p)] = (float(glr), float(gr.get("weight_decay", weight_decay)))
        if bucket is None:
            from .parallel import GradBucket
            bucket = GradBucket([p for gr in groups for p in gr["params"]])
        self.bucket = bucket
        self.params: List[torch.nn.Parameter] = bucket.params
        in_bucket = {id(p) for p in self.params}
        missing = [p for gr in groups for p in gr["params"] if p.requires_grad and id(p) not in in_bucket]
        if missing:
            # such parameters would silently never be updated and would be left out of the --gradclip norm
            raise ValueError("FlatBertAdam: %d trainable parameter(s) of the param groups (%d elements) are not in the "
                             "gradient bucket; build the GradBucket from the same parameters (e.g. GradBucket(p for g in "
                             "groups for p in g['params'])) or give those parameters to a second optimiser"
                             % (len(missing), sum(p.numel() for p in missing)))
        for p in self.params:
            if id(p) not in per:
                raise ValueError("FlatBertAdam: the gradient bucket holds a parameter that is in no param group")
            if not p.is_cuda or p.dtype != torch.float32:
                raise L.SxError("FlatBertAdam needs fp32 CUDA parameters (no CPU fallback)")
        dev = self.params[0].device
        # flat parameter buffer, same layout as the gradient bucket
        self.flat_p = torch.empty(bucket.numel, device=dev, dtype=torch.float32)
        self.flat_p.zero_()
        seg_param, seg_off, seg_len = [], [], []
        for i, (p, off) in enumerate(zip(self.params, bucket.offsets)):
            n = p.numel()
            view = self.flat_p[off:off + n].view_as(p)
            view.copy_(p.data)
            p.data = view
            for s in range(0, n, _SEG):
                seg_param.append(i)
                seg_off.append(off + s)
                seg_len.append(min(_SEG, n - s))
        # TF32-rounded twin of the parameters, kept current by the update kernel: ops.round_tf32(p) returns the view in
        # `p._sx_tf32` while p._version is unchanged, which removes the per-weight rounding pass from every forward.
        # (In-place edits through torch bump the version and fall back to rounding on the fly; after raw `.data` edits
        # call refresh_rounded().)
        self.flat_r = torch.empty_like(self.flat_p)
        self.refresh_rounded()
        self.flat_m = torch.zeros_like(self.flat_p)
        self.flat_v = torch.zeros_like(self.flat_p)
        P = len(self.params)
        self._seg_param = torch.tensor(seg_param, dtype=torch.int32, device=dev)
        self._seg_off = torch.tensor(seg_off, dtype=torch.int64, device=dev)
        self._seg_len = torch.tensor(seg_len, dtype=torch.int32, device=dev)
        self._lr = torch.tensor([per[id(p)][0] for p in self.params], dtype=torch.float32, device=dev)
        self._wd = torch.tensor([per[id(p)][1] for p in self.params], dtype=torch.float32, device=dev)
        self.step_count = torch.zeros(1, dtype=torch.int64, device=dev)          # device-resident
        self._sumsq = torch.empty(P, dtype=torch.float64, device=dev)
        self._coef = torch.empty(P, dtype=torch.float32, device=dev)
        self._lr_eff = torch.empty(P, dtype=torch.float32, device=dev)
        self.grad_norm = torch.zeros(1, dtype=torch.float32, device=dev)         # pre-clip global norm of the last step
        self.hyper = dict(b1=b1, b2=b2, e=e, max_grad_norm=max_grad_norm, grad_clip=grad_clip, warmup=warmup,
                          t_total=t_total, schedule=schedule)
        # torch.optim.Optimizer-shaped view of the configuration (what the reference's checkpoints and LR logging read)
        self.param_groups = []
        pos = {id(p): i for i, p in enumerate(self.params)}
        for gr in groups:
            glr = gr.get("lr", lr)
            self.param_groups.append({"params": [p for p in gr["params"] if id(p) in pos], "lr": float(glr),
                                      "weight_decay": float(gr.get("weight_decay", weight_decay)), "schedule": schedule,
                                      "warmup": warmup, "t_total": t_total, "b1": b1, "b2": b2, "e": e,
                                      "max_grad_norm": max_grad_norm})

    def refresh_rounded(self):
        L.call("sx_convert", self.flat_p.data_ptr(), L.SX_F32, self.flat_p.numel(), self.flat_r.data_ptr(), L.SX_F32, 1,
               ops._stream())
        for p, off in zip(self.params, self.bucket.offsets):
            p._sx_tf32 = self.flat_r[off:off + p.numel()].view_as(p)
            p._sx_tf32_version = p._version
            p._sx_tf32_ptr = p.data_ptr()

    def zero_grad(self, set_to_none: bool = False):
        """One memset of the bucket (the .grad views stay attached; set_to_none is ignored on purpose)."""
        self.bucket.zero()

    def step(self):
        h = self.hyper
        sched = L.SX_SCHED_WARMUP_LINEAR if h["schedule"] == "warmup_linear" else L.SX_SCHED_WARMUP_CONSTANT
        L.call("sx_adam_step", self.flat_p.data_ptr(), self.flat_r.data_ptr(), self.bucket.flat.data_ptr(), self.flat_m.data_ptr(),
               self.flat_v.data_ptr(), self._seg_param.data_ptr(), self._seg_off.data_ptr(), self._seg_len.data_ptr(),
               self._seg_param.numel(), len(self.params), self._lr.data_ptr(), self._wd.data_ptr(), h["b1"], h["b2"],
               h["e"], float(h["grad_clip"]), float(h["max_grad_norm"]), float(h["warmup"]), int(h["t_total"]), sched,
               self.step_count.data_ptr(), self._sumsq.data_ptr(), self._coef.data_ptr(), self._lr_eff.data_ptr(),
               self.grad_norm.data_ptr(), ops._stream())
        # the kernel has just rewritten the TF32 twin of EVERY parameter: twins invalidated by an in-place torch edit since
        # the last step (e.g. load_state_dict, which bumps the version counters) are valid again
        for p in self.params:
            if p._sx_tf32_version != p._version:
                p._sx_tf32_version = p._version

    def get_lr(self):
        """Scheduled learning rates of the LAST step (one device read; the reference's get_lr(), optimization.py:75-88)."""
        return self._lr_eff.tolist()

    def state_dict(self):
        """torch.optim.Optimizer layout (what the reference stores as 'optim_state', train3d.py:398): per-parameter
        {'step', 'next_m', 'next_v'} keyed by the parameter's index, plus the param_groups with index lists."""
        step = int(self.step_count.item())
        state, idx = {}, {id(p): i for i, p in enumerate(self.params)}
        for i, (p, off) in enumerate(zip(self.params, self.bucket.offsets)):
            n = p.numel()
            state[i] = {"step": step, "next_m": self.flat_m[off:off + n].view_as(p).clone(),
                        "next_v": self.flat_v[off:off + n].view_as(p).clone()}
        groups = [{k: (v if k != "params" else [idx[id(p)] for p in v]) for k, v in g.items()} for g in self.param_groups]
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd):
        """Accepts the layout above (also as written by the reference's BertAdam for the same parameter order) and the
        round-1 flat layout {'step', 'next_m', 'next_v'}."""
        if "state" in sd:
            st = sd["state"]
            if len(st) > len(self.params):
                raise ValueError("FlatBertAdam.load_state_dict: %d parameter states for %d parameters" % (len(st), len(self.params)))
            steps = set()
            for i, (p, off) in enumerate(zip(self.params, self.bucket.offsets)):
                e = st.get(i, st.get(str(i)))
                if e is None:                      # the reference keeps no state for parameters that never got a gradient
                    continue
                n = p.numel()
                if e["next_m"].numel() != n or e["next_v"].numel() != n:
                    raise ValueError("FlatBertAdam.load_state_dict: parameter %d has %d elements, the checkpoint %d"
                                     % (i, n, e["next_m"].numel()))
                self.flat_m[off:off + n].copy_(e["next_m"].reshape(-1))
                self.flat_v[off:off + n].copy_(e["next_v"].reshape(-1))
                steps.add(int(e["step"]))
            if steps:
                self.step_count.fill_(max(steps))
            for g_new, g_old in zip(self.param_groups, sd.get("param_groups", [])):
                for k in ("lr", "weight_decay"):
                    if k in g_old:
                        g_new[k] = float(g_old[k])
            pos = {id(p): i for i, p in enumerate(self.params)}
            for g in self.param_groups:
                for p in g["params"]:
                    self._lr[pos[id(p)]] = g["lr"]
                    self._wd[pos[id(p)]] = g["weight_decay"]
            return
        if sd["next_m"].numel() != self.flat_m.numel() or sd["next_v"].numel() != self.flat_v.numel():
            raise ValueError("FlatBertAdam.load_state_dict: flat moment buffers of %d elements expected, got %d"
                             % (self.flat_m.numel(), sd["next_m"].numel()))
        self.step_count.fill_(int(sd["step"]))
        self.flat_m.copy_(sd["next_m"])
        self.flat_v.copy_(sd["next_v"])
