"""Tensor-level operators of the hot path: thin wrappers that allocate outputs with torch, launch the
sm_90a kernels through the C ABI on torch's current stream, and wire them into autograd.

PyTorch is used for device memory, streams and the autograd tape only; every arithmetic step below is
one of the library's own kernels (no ATen math on the path, no fallbacks).
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import numpy as np
import torch

from . import _lib as L

# ------------------------------------------------------------------------------------------------
# precision policy
# ------------------------------------------------------------------------------------------------
# "tf32":   activations/weights stay fp32 in HBM, tensor cores consume them as TF32 (operands pre-rounded
#           to nearest so the hardware truncation is exact) with fp32 accumulation — parity-grade (<=1e-3).
# "bf16":   fast, NON-parity mode (BASELINE.json's "bf16 in, fp32 accum"; cfg 5): every contraction runs on the tensor
#           cores as kind::f16 with bf16 operands (2x the TF32 rate) and fp32 accumulation; tensors stay fp32 in HBM and
#           each GEMM operand is converted once (the bf16 copy is cached for its other uses in the step).  Statistics
#           (LayerNorm, softmax, GELU, aggregation), the head and the optimiser stay fp32.  Error budget: DESIGN §2.
# "tf32x3": validation mode.  No producer rounds; every GEMM runs as three TF32 passes on the split operands
#           (A_hi B_hi + A_lo B_hi + A_hi B_lo, fp32 accumulate), which recovers fp32-level products (~1e-6).
#           3x the tensor work plus the operand splits — used by the parity tests to show that the kernels and
#           the re-associated algebra are exact and TF32 operand rounding is the only deviation of the fast mode.
_PRECISION = "tf32"


def set_precision(p: str):
    global _PRECISION
    if p not in ("tf32", "tf32x3", "bf16"):
        raise ValueError("unsupported precision %r (this build implements 'tf32', 'tf32x3' and 'bf16')" % (p,))
    _PRECISION = p
    _bf16_cache.clear()


def get_precision() -> str:
    return _PRECISION


# Per-contraction precision policy of the default ("tf32") mode.  Every GEMM call site carries a tag:
#   "small": attractor-row and weight-space products (A rows or none: q1, Q1.Wk, the in-squeeze value projection, the
#            squeeze-out key projection, the folded value bank W' = Wm Wv and V' = a W'^T) — a few % of the FLOPs when
#            the attractor bank is small against the token count ("smallwide" otherwise, see small_tag);
#   "proj" : token-row projections (N rows x C x C: the squeeze-out query projection);
#   "insq" : the in-squeeze attention products (A x N x C);
#   "big"  : scores, P.V', the grouped output Linear and everything in backward that is their size.
# A tag mapped to "tf32x3" runs its FORWARD product as one launch over K-concatenated hi/lo operand splits (three TF32
# partial products, fp32-grade result); "tf32" is one pass on TF32-rounded operands; backward products are always single
# pass (gradients are held to 3e-3, not 1e-3).  The default keeps the small forward contractions exact: they feed every
# token through the attractor bank, so their rounding error is shared by all outputs; making the token-row projections or
# the in-squeeze products 3-pass as well does not change the full-size forward error.
_POLICY = {"small": "tf32x3", "smallwide": "tf32", "proj": "tf32", "insq": "tf32", "big": "tf32"}


def small_tag(rows_small: int, rows_tokens: int) -> str:
    """Precision class of an attractor-row / weight-space contraction: "small" (3-pass by default) while the attractor bank
    is at most a quarter of the token count — there its products are a few % of the layer's FLOPs (every 2-D BASELINE
    config: 256 attractors against 1296-5184 tokens) — and "smallwide" (single pass by default) when the bank is comparable
    to the token count (cfg 4/5: 1024 / 2048 attractors against 2744 / 5832 tokens, where these products are ~20 % of the
    FLOPs and the single-pass error is 4-7e-4 anyway)."""
    return "small" if 4 * int(rows_small) <= int(rows_tokens) else "smallwide"


def set_precision_policy(**kw):
    for k, v in kw.items():
        if k not in _POLICY or v not in ("tf32", "tf32x3"):
            raise ValueError("set_precision_policy: unknown tag/mode %s=%r" % (k, v))
        _POLICY[k] = v


def get_precision_policy():
    return dict(_POLICY)


def _three_pass(tag: str) -> bool:
    return _PRECISION == "tf32x3" or (_PRECISION == "tf32" and _POLICY.get(tag, "tf32") == "tf32x3")


def rt_for(tag: str) -> int:
    """round-to-TF32 flag for a producer whose output is consumed ONLY by contractions of class `tag`."""
    return 0 if _three_pass(tag) else 1


# Direct gradient accumulation (opt-in, used by parallel.GradBucket(direct_accumulate=True)): when a weight is a leaf
# whose .grad already exists (a view into the flat gradient bucket), the weight-gradient GEMM / bias column sum
# accumulates straight into it and autograd receives None for that input — this removes the zero-fill of a temporary
# and the AccumulateGrad add (two extra passes over every weight gradient).  Post-accumulate hooks do not fire.
_GRAD_SINK = False


def set_grad_sink(on: bool):
    global _GRAD_SINK
    _GRAD_SINK = bool(on)


# Gradient-ready milestones (parallel.GradBucket(milestones=True)): modules mark tensors at layer boundaries; when the
# backward pass reaches such a tensor every node created after it has already run (autograd executes in descending
# creation order), so the gradients of the parameters used after that point are final and their all-reduce can start.
_GRAD_READY_CB = None


def set_grad_ready_callback(fn):
    global _GRAD_READY_CB
    _GRAD_READY_CB = fn


def grad_ready(t: torch.Tensor, params):
    """When backward reaches `t`, announce that the gradients of `params` are final.  No-op without a callback.
    `t` must be the RESULT of an operation: its hook then runs as a pre-hook of the node that produced it, i.e. after every
    node created later AND after their (top-priority) AccumulateGrad nodes.  A leaf's hook sits on its own AccumulateGrad
    node, whose order against the AccumulateGrad nodes of sibling parameters is unspecified — leaves are therefore not
    marked (their parameters are covered by the final GradBucket.allreduce_async())."""
    if _GRAD_READY_CB is None or not isinstance(t, torch.Tensor) or not t.requires_grad or t.grad_fn is None:
        return
    ps = list(params)
    cb = _GRAD_READY_CB

    def hook(_g):
        cb(ps)
        return None

    t.register_hook(hook)


def _grad_target(p):
    if not _GRAD_SINK or not isinstance(p, torch.nn.Parameter) or p.grad is None:
        return None
    g = p.grad
    if g.dtype != torch.float32 or not g.is_contiguous() or g.shape != p.shape or not g.is_cuda:
        return None
    return g


def _sink_or_zeros(p, like=None):
    """-> (buffer the kernel accumulates into, gradient to hand to autograd or None when it went straight to p.grad)."""
    tgt = _grad_target(p)
    if tgt is not None:
        return tgt, None
    z = _zeros_like(p if like is None else like)
    return z, z


def _rt() -> int:
    """round-to-TF32 flag handed to producer kernels (off in the 3-pass validation mode)."""
    return 1 if _PRECISION == "tf32" else 0


# ------------------------------------------------------------------------------------------------
# dropout seeds (CUDA-graph safe): a per-device base seed lives on the GPU; every dropout site derives its own
# per-call device seed from it in stream order and keeps that tensor for backward, so a captured graph draws a
# fresh mask on every replay and fwd/bwd of one call always agree.
# ------------------------------------------------------------------------------------------------
_MASK64 = (1 << 64) - 1
_base_seeds = {}
_site_counter = [0]


def _base_seed(device) -> torch.Tensor:
    key = (device.type, device.index)
    t = _base_seeds.get(key)
    if t is None:
        t = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).to(device)       # follows torch.manual_seed
        _base_seeds[key] = t
    return t


def reseed(seed: int, device=None):
    """Set the dropout base seed explicitly (all devices, or one)."""
    for key, t in list(_base_seeds.items()):
        if device is None or (device.type, device.index) == key:
            t.fill_(int(seed) & ((1 << 62) - 1))


def advance_seed(device):
    """Bump the base seed once per training step (captured into CUDA graphs like any other kernel)."""
    L.call("sx_seed_advance", _base_seed(device).data_ptr(), 0xD1B54A32D192ED03, _stream())
    _begin_zero_arena(device)                   # step boundary: one memset for all zero-initialised scratch of the step
    _bf16_cache.clear()


def new_dropout_seed(device) -> torch.Tensor:
    """Per-call device seed = base seed + a unique site constant; pass it as `seed=` to a dropout-capable op."""
    _site_counter[0] += 1
    t = torch.empty(1, device=device, dtype=torch.int64)
    L.call("sx_seed_derive", _base_seed(device).data_ptr(), (_site_counter[0] * 0x9E3779B97F4A7C15) & _MASK64,
           t.data_ptr(), _stream())
    return t


def _seed_args(seed):
    """seed: python int (by value) or int64 device tensor (by pointer) -> (value, pointer)."""
    if isinstance(seed, torch.Tensor):
        return 0, seed.data_ptr()
    return int(seed) & _MASK64, None


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _req_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise L.SxError("segtran_b200 ops need CUDA tensors (no CPU fallback); got a %s tensor" % t.device)


# ------------------------------------------------------------------------------------------------
# zero-initialised scratch (accumulation targets of split-K / batch-reduced GEMMs and column sums): instead of one tiny
# fill kernel per buffer (~40 per training step), every request of a step is carved out of ONE arena that a single
# memset clears.  A new arena tensor is allocated at each step boundary (advance_seed), sized by the largest step seen so
# far; slices keep their arena alive, so nothing is ever recycled under a live tensor.  Outside of training steps (or on
# the first step) requests fall back to torch.zeros.
# ------------------------------------------------------------------------------------------------
_zero_arena = {}
_ARENA_MAX = 1 << 26          # floats (256 MB)


def _arena_state(device):
    return _zero_arena.setdefault((device.type, device.index), {"buf": None, "off": 0, "peak": 0})


def _begin_zero_arena(device):
    st = _arena_state(device)
    st["peak"] = max(st["peak"], st["off"])
    st["off"] = 0
    st["buf"] = torch.zeros(st["peak"], device=device, dtype=torch.float32) if st["peak"] else None


def _zeros(shape, device) -> torch.Tensor:
    if isinstance(shape, int):
        shape = (shape,)
    n = 1
    for d in shape:
        n *= int(d)
    st = _arena_state(device)
    off, n_al = st["off"], (n + 63) // 64 * 64           # 256-byte slots (TMA / vector accesses stay legal)
    # the running demand sizes the next arena; it is capped so that many forwards without a step boundary in between
    # (evaluation loops) cannot inflate it
    st["off"] = min(off + n_al, _ARENA_MAX)
    if st["buf"] is not None and off + n_al <= st["buf"].numel():
        return st["buf"][off:off + n].view(tuple(shape))
    return torch.zeros(tuple(shape), device=device, dtype=torch.float32)


def _zeros_like(t: torch.Tensor) -> torch.Tensor:
    return _zeros(tuple(t.shape), t.device)


# ------------------------------------------------------------------------------------------------
# GEMM on strided views:  C[..., m, n] = epilogue(alpha * sum_k A[..., m, k] B[..., n, k])
# ------------------------------------------------------------------------------------------------
def _operand(t: torch.Tensor, Z1: int, Z0: int, name: str) -> L.sx_operand:
    # t: [z1, z0, R, K] view (batch dims of size 1 broadcast)
    R, K = t.shape[-2], t.shape[-1]
    sr, sk = t.stride(-2), t.stride(-1)
    if sk == 1 or K == 1:
        major, ld = L.SX_MAJOR_K, sr
        if R == 1:
            ld = max(K, 4)
    elif sr == 1 or R == 1:
        major, ld = L.SX_MAJOR_MN, sk
    else:
        raise L.SxError("gemm operand %s: neither dim is contiguous (strides %s)" % (name, t.stride()))
    op = L.sx_operand()
    op.ptr = t.data_ptr()
    op.major = major
    op.ld = ld
    op.stride_z0 = t.stride(1) if t.shape[1] > 1 else 0
    op.stride_z1 = t.stride(0) if t.shape[0] > 1 else 0
    return op


def _as4(t: torch.Tensor) -> torch.Tensor:
    while t.dim() < 4:
        t = t.unsqueeze(0)
    if t.dim() != 4:
        raise L.SxError("gemm operands must have <= 4 dims")
    return t


# bf16 operand copies of the current step (precision "bf16"): key -> (source tensor kept alive, bf16 copy).  Holding the
# source keeps its storage from being recycled under a live key; the cache is emptied at every step boundary.
_bf16_cache = {}
_BF16_CACHE_MAX = 96


def _bf16_view(t4: torch.Tensor) -> torch.Tensor:
    """fp32 4-D operand view -> bf16 tensor with the same logical layout (element strides), converted once per step.
    The conversion is done on the view's whole underlying storage (one pass, shared by every other view of the same
    tensor: q/k/v mode slices, transposes, the forward and the backward uses); storages much larger than the view
    (slices of an arena) are converted per view."""
    st = t4.untyped_storage()
    n_st = st.nbytes() // 4
    if n_st <= 4 * t4.numel() + 1024 and st.data_ptr() % 16 == 0:
        key = ("st", st.data_ptr(), n_st, t4._version)
        hit = _bf16_cache.get(key)
        if hit is None:
            flat = torch.empty(n_st, device=t4.device, dtype=torch.bfloat16)
            L.call("sx_convert", st.data_ptr(), L.SX_F32, n_st, flat.data_ptr(), L.SX_BF16, 0, _stream())
            if len(_bf16_cache) >= _BF16_CACHE_MAX:
                _bf16_cache.pop(next(iter(_bf16_cache)))
            hit = (t4, flat)
            _bf16_cache[key] = hit
        return torch.as_strided(hit[1], t4.size(), t4.stride(), t4.storage_offset())
    key = (t4.data_ptr(), tuple(t4.shape), tuple(t4.stride()), t4._version)
    hit = _bf16_cache.get(key)
    if hit is not None:
        return hit[1]
    dims = sorted(((s_, z_) for s_, z_ in zip(t4.stride(), t4.shape) if z_ > 1), key=lambda x: x[0])
    dense, span = True, 1
    for s_, z_ in dims:
        dense = dense and s_ == span
        span *= z_
    src = t4 if dense else t4.contiguous()
    out = torch.empty_strided(src.size(), src.stride(), device=src.device, dtype=torch.bfloat16)
    L.call("sx_convert", src.data_ptr(), L.SX_F32, src.numel(), out.data_ptr(), L.SX_BF16, 0, _stream())
    if len(_bf16_cache) >= _BF16_CACHE_MAX:
        _bf16_cache.pop(next(iter(_bf16_cache)))
    _bf16_cache[key] = (t4, out)
    return out


_PART_FLOATS = 8 << 20          # 32 MB per (device, stream)
_part_bufs = {}


def _part_args(device):
    """(pointer, floats) of the scratch the library's ordered partial sums use (split-K partial tiles, per-CTA column
    sums).  One buffer per (device, stream): calls on one stream run in order, calls on different streams never share."""
    key = (device.index if device.index is not None else torch.cuda.current_device(), torch.cuda.current_stream(device).cuda_stream)
    t = _part_bufs.get(key)
    if t is None:
        t = _part_bufs[key] = torch.empty(_PART_FLOATS, device=device, dtype=torch.float32)
    return t.data_ptr(), t.numel()


def _pick_split_k(M, N, K, Z, bk=32, sms=132, epi=10):
    """Split-K factor for a GEMM whose 128 x 128 tile count does not fill the machine (132 SMs on an H100 SXM):
    minimise rounds(tiles*sk / SMs) * (k-blocks per unit + epilogue cost in k-block units)."""
    tiles = ((M + 127) // 128) * ((N + 127) // 128) * Z
    nkb = (K + bk - 1) // bk
    if tiles >= 2 * sms or nkb < 16:
        return 1
    best, best_cost = 1, None
    for sk in range(1, max(1, nkb // 8) + 1):
        rounds = (tiles * sk + sms - 1) // sms
        cost = rounds * ((nkb + sk - 1) // sk + epi * (1 if sk == 1 else 2))     # atomics make split epilogues dearer
        if best_cost is None or cost < best_cost:
            best, best_cost = sk, cost
    return best


def _gemm_nt_1(a: torch.Tensor, b: torch.Tensor, *, out: Optional[torch.Tensor] = None, alpha: float = 1.0,
               bias: Optional[torch.Tensor] = None, bias_mode: int = L.SX_BIAS_N, gelu: bool = False,
               preact: Optional[torch.Tensor] = None, accumulate: bool = False, split_k: Optional[int] = None,
               amax: Optional[torch.Tensor] = None, drop_p: float = 0.0, seed: int = 0, round_out: bool = True,
               reduce_z1: bool = False, addend: Optional[torch.Tensor] = None,
               gelu_bwd: Optional[torch.Tensor] = None, colsum: Optional[torch.Tensor] = None) -> torch.Tensor:
    """a [..., M, K], b [..., N, K] (strided fp32 views; either dim may be the contiguous one) ->
    out [z1, z0, M, N] fp32.  With reduce_z1 the z1 batch dim is summed into one output (atomic accumulate)."""
    _req_cuda(a, b, out, bias, preact, amax)
    if a.dtype != torch.float32 or b.dtype != torch.float32:
        raise L.SxError("gemm_nt: fp32 operands expected (precision policy %s)" % _PRECISION)
    a4, b4 = _as4(a), _as4(b)
    M, K = a4.shape[-2:]
    N, K2 = b4.shape[-2:]
    if K != K2:
        raise L.SxError("gemm_nt: K mismatch %d vs %d" % (K, K2))
    Z1 = max(a4.shape[0], b4.shape[0])
    Z0 = max(a4.shape[1], b4.shape[1])
    for t in (a4, b4):
        if t.shape[0] not in (1, Z1) or t.shape[1] not in (1, Z0):
            raise L.SxError("gemm_nt: batch dims do not broadcast")
    oz1 = 1 if reduce_z1 else Z1
    fresh = out is None
    linear_epi = (not gelu) and preact is None and drop_p == 0.0 and amax is None and gelu_bwd is None
    if split_k is None:
        split_k = _pick_split_k(M, N, K, Z0 * Z1) if (linear_epi and (fresh or accumulate or reduce_z1)) else 1
    if fresh:
        if accumulate or reduce_z1 or split_k > 1:
            out = _zeros((oz1, Z0, M, N), a.device)
        else:
            out = torch.empty((oz1, Z0, M, N), device=a.device, dtype=torch.float32)
    o4 = _as4(out)
    if o4.shape[-2:] != (M, N) or o4.stride(-1) != 1:
        raise L.SxError("gemm_nt: bad output view %s %s" % (tuple(o4.shape), o4.stride()))
    g = L.sx_gemm_args()
    g.op_dtype = L.SX_OP_TF32
    if _PRECISION == "bf16":
        a4, b4 = _bf16_view(a4), _bf16_view(b4)
        g.op_dtype = L.SX_OP_BF16
    g.M, g.N, g.K, g.Z0, g.Z1 = M, N, K, Z0, Z1
    g.A = _operand(a4, Z1, Z0, "A")
    g.B = _operand(b4, Z1, Z0, "B")
    g.C = o4.data_ptr()
    g.c_dtype = L.SX_F32
    # a split-K / accumulating launch adds partial sums in memory: rounding each partial to TF32 would leave a sum that is
    # NOT a TF32 value (the tensor core would then truncate it), so the rounding becomes a pass over the finished output
    round_after = round_out and _PRECISION == "tf32" and (split_k > 1 or accumulate or reduce_z1)
    g.round_tf32 = 1 if (round_out and _PRECISION == "tf32" and not round_after) else 0
    g.ldc = o4.stride(-2)
    g.c_stride_z0 = o4.stride(1) if o4.shape[1] > 1 else 0
    g.c_stride_z1 = 0 if reduce_z1 else (o4.stride(0) if o4.shape[0] > 1 else 0)
    g.alpha = alpha
    if bias is not None:
        b4b = bias
        while b4b.dim() < 3:
            b4b = b4b.unsqueeze(0)
        g.bias = bias.data_ptr()
        g.bias_mode = bias_mode
        g.bias_stride_z0 = b4b.stride(1) if b4b.shape[1] > 1 else 0
        g.bias_stride_z1 = b4b.stride(0) if b4b.shape[0] > 1 else 0
    g.act = L.SX_ACT_GELU if gelu else L.SX_ACT_NONE
    if gelu_bwd is not None:                 # C = dropmask * (A.B^T) * gelu'(h): h (C's layout) goes in through `preact`
        if gelu or preact is not None or tuple(gelu_bwd.shape[-2:]) != (M, N) or gelu_bwd.stride() != out.stride():
            raise L.SxError("gemm_nt: gelu_bwd needs the pre-activation in the output's layout and no other activation")
        g.act = L.SX_ACT_GELU_BWD
        g.preact = gelu_bwd.data_ptr()
    g.split_k = split_k
    if split_k > 1:
        g.part, g.part_floats = _part_args(a.device)
    g.accumulate = 1 if (accumulate or reduce_z1 or split_k > 1) else 0
    if preact is not None:
        g.preact = preact.data_ptr()
    if amax is not None:
        g.amax = amax.data_ptr()
    g.drop_p = drop_p
    g.drop_seed, g.drop_seed_dev = _seed_args(seed)
    if colsum is not None:
        if colsum.dtype != torch.float32 or colsum.numel() != N or not colsum.is_contiguous() or accumulate or reduce_z1:
            raise L.SxError("gemm_nt: colsum must be a contiguous fp32 [N] tensor, without accumulate / reduce_z1")
    if addend is not None:
        if addend.dtype != torch.float32 or tuple(addend.shape[-2:]) != (M, N) or _as4(addend).stride() != o4.stride():
            raise L.SxError("gemm_nt: addend must be an fp32 tensor in the output's layout")
        g.addend = addend.data_ptr()
    L.call("sx_gemm", C.byref(g), _stream())
    if colsum is not None:                   # column sums of the stored values, in a fixed order (sx_colsum)
        o2 = o4.view(-1, N)
        L.call("sx_colsum", o2.data_ptr(), L.SX_F32, o2.shape[0], N, o2.stride(0), colsum.data_ptr(), *_part_args(o2.device), _stream())
    if round_after and fresh:                # (caller-provided accumulators are gradient buffers: never rounded)
        L.call("sx_convert", out.data_ptr(), L.SX_F32, out.numel(), out.data_ptr(), L.SX_F32, 1, _stream())
    return out


def gemm_nt(a: torch.Tensor, b: torch.Tensor, *, out: Optional[torch.Tensor] = None, alpha: float = 1.0,
            bias: Optional[torch.Tensor] = None, bias_mode: int = L.SX_BIAS_N, gelu: bool = False,
            preact: Optional[torch.Tensor] = None, accumulate: bool = False, split_k: Optional[int] = None,
            amax: Optional[torch.Tensor] = None, drop_p: float = 0.0, seed: int = 0, round_out: bool = True,
            reduce_z1: bool = False, gelu_bwd: Optional[torch.Tensor] = None,
            addend: Optional[torch.Tensor] = None, colsum: Optional[torch.Tensor] = None,
            tag: str = "big") -> torch.Tensor:
    """C[..., m, n] = epilogue(alpha * sum_k a[..., m, k] b[..., n, k]) on the wgmma GEMM.  One launch on TF32-rounded
    operands, or — in 'tf32x3' mode / for call-site classes the precision policy maps to it — three passes on the hi/lo
    operand splits (fp32-grade products)."""
    if not _three_pass(tag):
        return _gemm_nt_1(a, b, out=out, alpha=alpha, bias=bias, bias_mode=bias_mode, gelu=gelu, preact=preact,
                          accumulate=accumulate, split_k=split_k, amax=amax, drop_p=drop_p, seed=seed,
                          round_out=round_out, reduce_z1=reduce_z1, gelu_bwd=gelu_bwd, addend=addend, colsum=colsum)
    _req_cuda(a, b)
    # ONE launch over K-concatenated operand splits: [A_hi | A_lo | A_hi] . [B_hi | B_hi | B_lo]^T (fp32 accumulation in registers
    # over the three partial products), so every epilogue / accumulate / split-K option works unchanged
    return _gemm_nt_1(_split_cat(a, 0), _split_cat(b, 1), out=out, alpha=alpha, bias=bias, bias_mode=bias_mode, gelu=gelu,
                      preact=preact, accumulate=accumulate, split_k=split_k, amax=amax, drop_p=drop_p, seed=seed,
                      round_out=round_out, reduce_z1=reduce_z1, gelu_bwd=gelu_bwd, addend=addend, colsum=colsum)


def _split_cat(t: torch.Tensor, role: int) -> torch.Tensor:
    """[..., R, K] fp32 view (any strides) -> contiguous [z1, z0, R, 3*pad4(K)] K-concatenated TF32 split (see sx_split_tf32_cat)."""
    t4 = _as4(t)
    Z1, Z0, R, K = t4.shape
    Kp = _pad4(K)
    out = torch.empty((Z1, Z0, R, 3 * Kp), device=t.device, dtype=torch.float32)
    L.call("sx_split_tf32_cat", t4.data_ptr(), Z1, Z0, R, K, t4.stride(0), t4.stride(1), t4.stride(2), t4.stride(3), Kp, role,
           out.data_ptr(), _stream())
    return out


def _pad4(n: int) -> int:
    return (n + 3) // 4 * 4


def _rowpad_empty(shape, device) -> torch.Tensor:
    """[..., R, L] view whose row stride is padded to a multiple of 4 floats (TMA needs 16-byte row pitches)."""
    Lr = shape[-1]
    buf = torch.empty(tuple(shape[:-1]) + (_pad4(Lr),), device=device, dtype=torch.float32)
    return buf[..., :Lr]


def _rows_ok(t: torch.Tensor) -> bool:
    """rows contiguous, 16-byte row pitch, and leading dims dense on top of that pitch."""
    if t.stride(-1) != 1 or t.stride(-2) % 4 != 0 or t.data_ptr() % 16 != 0:
        return False
    exp = t.stride(-2) * t.shape[-2]
    for d in range(t.dim() - 3, -1, -1):
        if t.shape[d] > 1 and t.stride(d) != exp:
            return False
        exp *= t.shape[d]
    return True


def _rowpad(t: torch.Tensor) -> torch.Tensor:
    if _rows_ok(t):
        return t
    o = _rowpad_empty(t.shape, t.device)
    o.copy_(t)
    return o


def round_tf32(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> fp32 rounded to the nearest TF32 value (weights, once per step)."""
    _req_cuda(x)
    if _PRECISION == "tf32":
        # parameters managed by train.FlatBertAdam carry a TF32-rounded twin that the optimiser kernel keeps current
        # (`_sx_tf32`); it is valid as long as nobody modified the parameter in place since (version counter)
        r = getattr(x, "_sx_tf32", None)
        if r is not None and getattr(x, "_sx_tf32_version", -1) == x._version and \
                getattr(x, "_sx_tf32_ptr", None) == x.data_ptr():
            return r
    x = x.contiguous()
    if _PRECISION != "tf32":
        return x
    y = torch.empty_like(x)
    L.call("sx_convert", x.data_ptr(), L.SX_F32, x.numel(), y.data_ptr(), L.SX_F32, 1, _stream())
    return y


def colsum(x2d: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[c] += sum_r x2d[r, c] (rows uniformly strided)."""
    if out is None:
        out = _zeros((x2d.shape[1],), x2d.device)
    L.call("sx_colsum", x2d.data_ptr(), L.SX_F32, x2d.shape[0], x2d.shape[1], x2d.stride(0), out.data_ptr(), *_part_args(x2d.device), _stream())
    return out


# ------------------------------------------------------------------------------------------------
# autograd functions
# ------------------------------------------------------------------------------------------------
class _Linear(torch.autograd.Function):
    """y = dropout(act(x W^T + b)).  nn.Linear call sites segtran_shared.py:243, :414, :559-560.  `tag` = precision class
    of the three products (forward, dx, dW), see the precision policy above."""

    @staticmethod
    def forward(ctx, x, W, b, gelu, drop_p, seed, tag, round_y):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        Wr = W.contiguous() if _three_pass(tag) else round_tf32(W)
        O = W.shape[0]
        y = torch.empty((x2.shape[0], O), device=x.device, dtype=torch.float32)
        h = torch.empty_like(y) if gelu else None
        gemm_nt(x2, Wr, out=y, bias=b, gelu=gelu, preact=h, drop_p=drop_p, seed=seed, tag=tag, round_out=round_y)
        ctx.save_for_backward(x2, Wr, h)
        ctx.meta = (shp, b is not None, gelu, drop_p, seed, tag)
        ctx.leaves = (W, b)
        return y.view(*shp[:-1], O)

    @staticmethod
    def backward(ctx, dy):
        x2, Wr, h = ctx.saved_tensors
        shp, has_b, gelu, drop_p, seed, tag = ctx.meta
        W, b = ctx.leaves
        if _three_pass(tag) and _PRECISION == "tf32":       # 3-pass forward, single-pass backward: TF32-rounded weight
            Wr = round_tf32(W)
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        if gelu:
            dh = torch.empty_like(dy2)
            L.call("sx_gelu_bwd", dy2.data_ptr(), h.data_ptr(), L.SX_F32, dy2.numel(), drop_p, *_seed_args(seed), dh.data_ptr(),
                   L.SX_F32, _rt(), _stream())
            dy2 = dh
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            dx = gemm_nt(dy2, Wr.t(), round_out=False).view(shp)
        if ctx.needs_input_grad[1]:
            tgt = _grad_target(W)
            if tgt is not None:
                gemm_nt(dy2.t(), x2.t(), out=tgt, accumulate=True, round_out=False)
            else:
                dW = gemm_nt(dy2.t(), x2.t(), round_out=False).view(Wr.shape)
        if has_b and ctx.needs_input_grad[2]:
            tgt = _grad_target(b)
            if tgt is not None:
                colsum(dy2, out=tgt)
            else:
                db = colsum(dy2)
        return dx, dW, db, None, None, None, None, None


def linear(x, W, b=None, gelu=False, drop_p=0.0, seed=0, tag="big", round_out=True):
    """round_out: round y to TF32 (set False when every consumer of y is a 3-pass contraction or not a GEMM)."""
    return _Linear.apply(x, W, b, gelu, drop_p, seed, tag, round_out)


class _AttnScores(torch.autograd.Function):
    """S[b,m] = scale * Q[b,:,m] K[b,:,m]^T (+ row_bias[u1])   (segtran_shared.py:566-567); tracks max(S) on the device.
    q may have batch 1 (the batch-invariant attractor queries): it is broadcast, and its gradient reduced over b.
    row_bias [U1] (single-mode only) is the per-query constant of the re-associated in-squeeze (see
    SqueezedAttFeatTrans): it is added after the scaling, so it must already be scaled."""

    @staticmethod
    def forward(ctx, q, k, M, amax, row_bias, tag, alpha=None):
        Bq, U1, Cq = q.shape
        B, U2 = k.shape[0], k.shape[1]
        d = Cq // M
        scale = 1.0 / math.sqrt(d) if alpha is None else float(alpha)
        qv = q.view(Bq, U1, M, d).permute(0, 2, 1, 3)         # [Bq,M,U1,d] strided view, d contiguous
        kv = k.view(B, U2, M, d).permute(0, 2, 1, 3)
        S = _rowpad_empty((B, M, U1, U2), q.device)
        if row_bias is not None and M != 1:
            raise L.SxError("attn_scores: row_bias needs a single mode")
        rb = row_bias.contiguous().view(-1) if row_bias is not None else None
        gemm_nt(qv, kv, out=S, alpha=scale, amax=amax, round_out=False, bias=rb, bias_mode=L.SX_BIAS_M, tag=tag)
        ctx.save_for_backward(q, k)
        ctx.meta = (M, d, scale, row_bias.shape if row_bias is not None else None)
        ctx.tag = tag
        return S

    @staticmethod
    def backward(ctx, dS):
        q, k = ctx.saved_tensors
        M, d, scale, rb_shape = ctx.meta
        Bq, U1, Cq = q.shape
        B, U2 = k.shape[0], k.shape[1]
        dS = _rowpad(dS)
        dq, dk = _score_grads(dS, q, k, M, scale, ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.tag)
        drb = None
        if rb_shape is not None and ctx.needs_input_grad[4]:
            drb = _zeros((U1,), q.device)     # sum over batch and keys
            L.call("sx_rowsum", dS.data_ptr(), B * U1, U2, dS.stride(-2), U1, drb.data_ptr(), *_part_args(dS.device), _stream())
            drb = drb.view(rb_shape)
        return dq, dk, None, None, drb, None, None


def _score_grads(dS, q, k, M, scale, need_q, need_k, tag="big"):
    """Gradients of S = scale * Q K^T per mode: dQ = scale dS K, dK = scale dS^T Q (q may have batch 1: broadcast)."""
    Bq, U1, Cq = q.shape
    B, U2 = k.shape[0], k.shape[1]
    d = Cq // M
    dq = dk = None
    if need_q:
        # dQ[b,m] (U1 x d) = scale * dS[b,m] (U1 x U2) . K[b,m] (U2 x d)
        bcast = Bq == 1 and B > 1
        dq = _zeros_like(q) if bcast else torch.empty_like(q)
        gemm_nt(dS, k.view(B, U2, M, d).permute(0, 2, 3, 1), out=dq.view(Bq, U1, M, d).permute(0, 2, 1, 3),
                alpha=scale, round_out=False, reduce_z1=bcast, split_k=1, tag=tag)
    if need_k:
        dk = torch.empty_like(k)
        gemm_nt(dS.transpose(-1, -2), q.view(Bq, U1, M, d).permute(0, 2, 3, 1),
                out=dk.view(B, U2, M, d).permute(0, 2, 1, 3), alpha=scale, round_out=False, tag=tag)
    return dq, dk


class PosBias:
    """Sliding-window positional bias of a self-attention (SlidingPosBiases2D/3D, segtran_shared.py:1002-1175) without
    the [N,N] matrix: token n is cell n of the row-major grid `grid` (2 or 3 extents), and the score of query q and key k
    gains w * table[k - q + R] (per dimension) when k lies within R cells of q in every dimension, 0 otherwise.
    table [2R+1]^pd is the learned parameter (or an eval-mode snapshot of it); w is pos_code_weight."""
    __slots__ = ("table", "R", "grid", "w")

    def __init__(self, table, R, grid, w=1.0):
        grid = tuple(int(g) for g in grid)
        if len(grid) not in (2, 3) or table.dim() != len(grid) or any(s != 2 * R + 1 for s in table.shape):
            raise L.SxError("PosBias: table %s does not match radius %d over grid %s" % (tuple(table.shape), R, grid))
        self.table, self.R, self.grid, self.w = table, int(R), grid, float(w)

    def with_weight(self, w):
        return PosBias(self.table, self.R, self.grid, w)

    @property
    def num_tokens(self):
        n = 1
        for g in self.grid:
            n *= g
        return n


def _posbias_desc(table, R, grid, w) -> L.sx_posbias:
    d = L.sx_posbias()
    d.table = table.data_ptr()
    d.pd, d.R = len(grid), R
    for i, g in enumerate(grid):
        d.grid[i] = g
    d.w = w
    return d


def _posbias_table(pb):
    t = pb.table
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise L.SxError("positional-bias table must be contiguous fp32")
    _req_cuda(t)
    return t


def attn_probs_fused(q, k, M, clip=500.0, drop_p=0.0, seed=0, diag=None, need_scores=False, round_out=True, posbias=None,
                     alpha=None):
    """P = dropout(softmax(min(Q K^T / sqrt(d), clip))) per mode in ONE wgmma kernel (csrc/sx_attn.cu): the scores stay
    in registers and the softmax runs on the accumulator fragments (reference segtran_shared.py:566-567, :569-580, :601, :605).
    q [Bq,U1,M*d] (Bq = 1 broadcasts), k [B,U2,M*d], both contiguous fp32 (TF32-rounded by their producers).
    posbias (PosBias, self-attention only): adds the sliding-window bias inside the softmax, after the clamp; S, rowmax
    and the clamp statistics stay on the raw scores (its table gradient comes from softmax_posbias_backward).
    alpha: the score scale (default 1/sqrt(d) of the per-mode width; the mince transformer scales zero-padded channel
    windows by the full width).
    -> (P [B,M,U1,U2] view of a row-padded buffer, S or None (raw scaled scores, same layout), lse [B,M,U1],
        rowmax [B,M,U1], stat [2])."""
    _req_cuda(q, k)
    if q.dtype != torch.float32 or k.dtype != torch.float32 or not q.is_contiguous() or not k.is_contiguous():
        raise L.SxError("attn_probs_fused: contiguous fp32 q/k expected")
    Bq, U1, Cq = q.shape
    B, U2, Ck = k.shape
    if Cq != Ck or Cq % M or (Cq // M) % 4 or Bq not in (1, B):
        raise L.SxError("attn_probs_fused: bad shapes q %s k %s modes %d" % (tuple(q.shape), tuple(k.shape), M))
    d = Cq // M
    P = _rowpad_empty((B, M, U1, U2), q.device)
    S = _rowpad_empty((B, M, U1, U2), q.device) if need_scores else None
    lse = torch.empty((B, M, U1), device=q.device, dtype=torch.float32)
    rowmax = torch.empty((B, M, U1), device=q.device, dtype=torch.float32)
    stat = _zeros((3,), q.device)
    a = L.sx_attn_probs_args()
    a.B, a.M, a.U1, a.U2, a.d = B, M, U1, U2, d
    a.round_tf32 = 1 if (round_out and _PRECISION == "tf32") else 0
    a.Q, a.q_ld, a.q_bstride = q.data_ptr(), Cq, (0 if Bq == 1 else U1 * Cq)
    a.K, a.k_ld, a.k_bstride = k.data_ptr(), Ck, U2 * Ck
    a.alpha, a.clip = (1.0 / math.sqrt(d) if alpha is None else float(alpha)), float(clip)
    a.P, a.S, a.ldp = P.data_ptr(), _ptr(S), P.stride(-2)
    a.lse, a.rowmax, a.stat, a.diag = lse.data_ptr(), rowmax.data_ptr(), stat.data_ptr(), _ptr(diag)
    a.drop_p = drop_p
    a.drop_seed, a.drop_seed_dev = _seed_args(seed)
    if posbias is not None:
        a.posbias = _posbias_desc(_posbias_table(posbias), posbias.R, posbias.grid, posbias.w)
    L.call("sx_attn_probs_fwd", C.byref(a), _stream())
    return P, S, lse, rowmax, stat


class _Scale(torch.autograd.Function):
    """y = alpha * x (sx_scale kernel)."""

    @staticmethod
    def forward(ctx, x, alpha):
        x = x.contiguous()
        y = torch.empty_like(x)
        L.call("sx_scale", x.data_ptr(), x.numel(), None, alpha, y.data_ptr(), _stream())
        ctx.alpha = alpha
        return y

    @staticmethod
    def backward(ctx, dy):
        return _Scale.apply(dy, ctx.alpha), None


def scale(x, alpha):
    return _Scale.apply(x, float(alpha))


class _Add(torch.autograd.Function):
    """y = a + b (same shapes)."""

    @staticmethod
    def forward(ctx, a, b):
        a, b = a.contiguous(), b.contiguous()
        y = torch.empty_like(a)
        L.call("sx_add", a.data_ptr(), b.data_ptr(), a.numel(), y.data_ptr(), _stream())
        return y

    @staticmethod
    def backward(ctx, dy):
        return dy, dy


def add(a, b):
    return _Add.apply(a, b)


class _MatVec(torch.autograd.Function):
    """y[r] = sum_c x[r,c] v[c] on CUDA cores (exact fp32; a K=1 / N=1 product has no business on tensor cores)."""

    @staticmethod
    def forward(ctx, x, v):
        x = x.contiguous()
        v = v.contiguous()
        R, Cd = x.shape
        y = _sgemm(x, v, R, 1, Cd, (Cd, 1), (1, 1))[0].view(R)
        ctx.save_for_backward(x, v)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, v = ctx.saved_tensors
        R, Cd = x.shape
        dy = dy.contiguous()
        dx = _sgemm(dy, v, R, Cd, 1, (1, 1), (1, 1))[0] if ctx.needs_input_grad[0] else None       # dy v^T
        dv = _sgemm(dy, x, 1, Cd, R, (1, 1), (Cd, 1))[0].view(Cd) if ctx.needs_input_grad[1] else None  # x^T dy
        return dx, dv


def matvec(x, v):
    return _MatVec.apply(x, v)


class _Softmax(torch.autograd.Function):
    """P = dropout(softmax(clamp_if(S)))  (segtran_shared.py:578-580, :601-605); output rounded for the P.V GEMM."""

    @staticmethod
    def forward(ctx, S, amax, clip, drop_p, seed, diag):
        S = _rowpad(S)
        Lr, ld = S.shape[-1], S.stride(-2)
        R = S.numel() // Lr
        P = _rowpad_empty(S.shape, S.device)
        lse = torch.empty(R, device=S.device, dtype=torch.float32)
        L.call("sx_softmax_fwd", S.data_ptr(), R, Lr, ld, _ptr(amax), clip, drop_p, *_seed_args(seed), P.data_ptr(), L.SX_F32,
               P.stride(-2), _rt(), lse.data_ptr(), _ptr(diag), _stream())
        ctx.save_for_backward(S, lse, amax)
        ctx.meta = (clip, drop_p, seed, P.stride(-2))
        return P

    @staticmethod
    def backward(ctx, dP):
        S, lse, amax = ctx.saved_tensors
        clip, drop_p, seed, ldp = ctx.meta
        dP = _rowpad(dP)
        Lr = S.shape[-1]
        R = S.numel() // Lr
        dS = _rowpad_empty(S.shape, S.device)
        L.call("sx_softmax_bwd", dP.data_ptr(), dP.stride(-2), S.data_ptr(), S.stride(-2), lse.data_ptr(), R, Lr,
               _ptr(amax), clip, drop_p, *_seed_args(seed), ldp, dS.data_ptr(), L.SX_F32, dS.stride(-2), _rt(), _stream())
        return dS, None, None, None, None, None


def softmax_posbias_backward(dP, ldd, S, lds, lse, R, Lr, amax, clip, drop_p, seed, ldp_fwd, dS, ldo, table, pb_geom,
                             table_needs_grad):
    """dS (with the clamp mask) and the table gradient of the biased softmax.  The table gradient goes straight into the
    table's .grad when direct accumulation is on (returns None then), else into a new tensor that is returned."""
    R_, grid, w = pb_geom
    tgt = _grad_target(table) if table_needs_grad else None
    buf = tgt if tgt is not None else _zeros((table.numel(),), table.device)
    desc = _posbias_desc(table, R_, grid, w)
    L.call("sx_softmax_posbias_bwd", dP.data_ptr(), ldd, S.data_ptr(), lds, lse.data_ptr(), R, Lr, _ptr(amax), clip, drop_p,
           *_seed_args(seed), ldp_fwd, dS.data_ptr(), L.SX_F32, ldo, _rt(), C.byref(desc), buf.data_ptr(),
           *_part_args(dS.device), _stream())
    if tgt is not None or not table_needs_grad:
        return None
    return buf.view(table.shape)


class _SoftmaxPosBias(torch.autograd.Function):
    """P = dropout(softmax(clamp_if(S) + w * bias))  (segtran_shared.py:578-605 with pos_biases); S is the raw [B,M,N,N]
    score tensor of a self-attention over the bias grid.  Backward: dS and the table gradient."""

    @staticmethod
    def forward(ctx, S, amax, clip, drop_p, seed, diag, table, pb_geom):
        S = _rowpad(S)
        Lr, ld = S.shape[-1], S.stride(-2)
        R = S.numel() // Lr
        P = _rowpad_empty(S.shape, S.device)
        lse = torch.empty(R, device=S.device, dtype=torch.float32)
        desc = _posbias_desc(table, *pb_geom)
        L.call("sx_softmax_posbias_fwd", S.data_ptr(), R, Lr, ld, _ptr(amax), clip, drop_p, *_seed_args(seed), P.data_ptr(),
               L.SX_F32, P.stride(-2), _rt(), lse.data_ptr(), _ptr(diag), C.byref(desc), _stream())
        ctx.save_for_backward(S, lse, amax, table)
        ctx.meta = (clip, drop_p, seed, P.stride(-2), pb_geom)
        ctx.leaf = table
        return P

    @staticmethod
    def backward(ctx, dP):
        S, lse, amax, table = ctx.saved_tensors
        clip, drop_p, seed, ldp, pb_geom = ctx.meta
        dP = _rowpad(dP)
        Lr = S.shape[-1]
        R = S.numel() // Lr
        dS = _rowpad_empty(S.shape, S.device)
        dT = softmax_posbias_backward(dP, dP.stride(-2), S, S.stride(-2), lse, R, Lr, amax, clip, drop_p, seed, ldp, dS,
                                      dS.stride(-2), ctx.leaf, pb_geom, ctx.needs_input_grad[6])
        return dS, None, None, None, None, None, dT, None


class _AttnPV(torch.autograd.Function):
    """U[b,m] = P[b,m] V[b,:,m]   with V [B,U2,M*F], channel = m*F+f  (segtran_shared.py:414-419, :447)."""

    @staticmethod
    def forward(ctx, P, v, M, tag, round_out):
        B, _, U1, U2 = P.shape
        Fd = v.shape[-1] // M
        vv = v.view(B, U2, M, Fd).permute(0, 2, 3, 1)          # [B,M,F,U2]: the "N x K" operand, F contiguous
        P = _rowpad(P)
        U = torch.empty((B, M, U1, Fd), device=P.device, dtype=torch.float32)
        gemm_nt(P, vv, out=U, tag=tag, round_out=round_out)
        ctx.save_for_backward(P, v)
        ctx.meta = (M, Fd)
        ctx.tag = tag
        return U

    @staticmethod
    def backward(ctx, dU):
        P, v = ctx.saved_tensors
        M, Fd = ctx.meta
        B, _, U1, U2 = P.shape
        dU = dU.contiguous()
        dP = dv = None
        if ctx.needs_input_grad[0]:
            # dP[b,m] (U1 x U2) = dU[b,m] (U1 x F) . V[b,m]^T  -> operand "B" = V[b,m] as [U2, F]
            dP = _rowpad_empty((B, M, U1, U2), P.device)
            gemm_nt(dU, v.view(B, U2, M, Fd).permute(0, 2, 1, 3), out=dP, round_out=False, tag=ctx.tag)
        if ctx.needs_input_grad[1]:
            dv = torch.empty_like(v)
            # dV[b,m] (U2 x F) = P[b,m]^T (U2 x U1) . dU[b,m] (U1 x F)
            gemm_nt(P.transpose(-1, -2), dU.transpose(-1, -2), out=dv.view(B, U2, M, Fd).permute(0, 2, 1, 3),
                    round_out=False, tag=ctx.tag)
        return dP, dv, None, None, None


class _AttnPVGelu(torch.autograd.Function):
    """G[b,m] = dropout(gelu(P[b,m] V'[b,:,m] + bias)) — the P.V contraction with MMSharedMid's bias / erf-GELU /
    dropout fused into its epilogue.  V' = V Wm^T is the value bank already pushed through the shared mid Linear
    (re-association (P V) Wm^T = P (V Wm^T): A rows instead of N, see ExpandedFeatTrans.forward)."""

    @staticmethod
    def forward(ctx, P, v, M, bias, drop_p, seed):
        B, _, U1, U2 = P.shape
        Fd = v.shape[-1] // M
        P = _rowpad(P)
        vv = v.view(B, U2, M, Fd).permute(0, 2, 3, 1)
        G = torch.empty((B, M, U1, Fd), device=P.device, dtype=torch.float32)
        H = torch.empty_like(G)
        gemm_nt(P, vv, out=G, bias=bias, gelu=True, preact=H, drop_p=drop_p, seed=seed)
        ctx.save_for_backward(P, v, H)
        ctx.meta = (M, Fd, drop_p, bias is not None)
        ctx.seed = seed
        return G

    @staticmethod
    def backward(ctx, dG):
        P, v, H = ctx.saved_tensors
        M, Fd, drop_p, has_b = ctx.meta
        B, _, U1, U2 = P.shape
        dG = dG.contiguous()
        dH = torch.empty_like(dG)
        L.call("sx_gelu_bwd", dG.data_ptr(), H.data_ptr(), L.SX_F32, dG.numel(), drop_p, *_seed_args(ctx.seed),
               dH.data_ptr(), L.SX_F32, _rt(), _stream())
        dP = dv = db = None
        if ctx.needs_input_grad[0]:
            dP = _rowpad_empty((B, M, U1, U2), P.device)
            gemm_nt(dH, v.view(B, U2, M, Fd).permute(0, 2, 1, 3), out=dP, round_out=False)
        if ctx.needs_input_grad[1]:
            dv = torch.empty_like(v)
            gemm_nt(P.transpose(-1, -2), dH.transpose(-1, -2), out=dv.view(B, U2, M, Fd).permute(0, 2, 1, 3),
                    round_out=False)
        if has_b and ctx.needs_input_grad[3]:
            db = colsum(dH.view(-1, Fd))
        return dP, dv, None, db, None, None


class _FoldedValueBank(torch.autograd.Function):
    """V'[b,a,m*F+o] = sum_f Wm[o,f] (a[b] Wv[m*F+f,:]^T) = a[b] . W'[m*F+o,:],  W'_m = Wm Wv_m   (segtran_shared.py:414 then
    :243 applied to the attractor rows, see ExpandedFeatTrans.forward): the value projection and MMSharedMid's Linear
    folded into ONE weight-space product (M F^2 C MACs, batch-independent) and ONE projection of the A attractor rows."""

    @staticmethod
    def forward(ctx, a, Wv, Wm, M, tag):
        B, A, Cd = a.shape
        Fd = Wm.shape[0]
        a2 = a.reshape(B * A, Cd)
        if not a2.is_contiguous():
            a2 = a2.contiguous()
        x3 = _three_pass(tag)
        Wvr = (Wv.contiguous() if x3 else round_tf32(Wv)).view(M, 1, Fd, Cd)      # [m, f, c]
        Wmr = Wm.contiguous() if x3 else round_tf32(Wm)                           # [o, f]
        # W'_m = Wm Wv_m [M,1,F(o),C]: kept unrounded when the bank projection below runs as a 3-pass product
        Wf = gemm_nt(Wmr.view(1, 1, Fd, Fd), Wvr.transpose(-1, -2), tag=tag, round_out=not x3)
        Vp = gemm_nt(a2, Wf.view(M * Fd, Cd), tag=tag)[0, 0]      # [B*A, M*F], TF32-rounded: the P.V' operand
        if x3 and _PRECISION == "tf32":                               # single-pass backward: TF32-rounded operands
            Wf, Wvr, Wmr = round_tf32(Wf), round_tf32(Wv).view(M, 1, Fd, Cd), round_tf32(Wm)
        ctx.save_for_backward(a2, Wf, Wvr, Wmr)
        ctx.meta = (B, A, Cd, Fd, M, Wv.shape)
        ctx.leaves = (Wv, Wm)
        return Vp.view(B, A, M * Fd)

    @staticmethod
    def backward(ctx, dVp):
        a2, Wf, Wvr, Wmr = ctx.saved_tensors
        B, A, Cd, Fd, M, wv_shape = ctx.meta
        Wv, Wm = ctx.leaves
        d2 = dVp.reshape(B * A, M * Fd)
        if not d2.is_contiguous():
            d2 = d2.contiguous()
        da = dWv = dWm = None
        if ctx.needs_input_grad[0]:
            da = gemm_nt(d2, Wf.view(M * Fd, Cd).t(), round_out=False)[0, 0].view(B, A, Cd)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dWf = gemm_nt(d2.t(), a2.t(), round_out=False).view(M, 1, Fd, Cd)          # [m, o, c]
            if ctx.needs_input_grad[2]:                               # dWm[o,f] = sum_m dW'_m[o,:] . Wv_m[f,:]
                tgt = _grad_target(Wm)
                if tgt is not None:
                    gemm_nt(dWf, Wvr, out=tgt.view(1, 1, Fd, Fd), reduce_z1=True, accumulate=True, round_out=False)
                else:
                    dWm = gemm_nt(dWf, Wvr, reduce_z1=True, round_out=False).view(Fd, Fd)
            if ctx.needs_input_grad[1]:                               # dWv_m[f,c] = sum_o Wm[o,f] dW'_m[o,c]
                tgt = _grad_target(Wv)
                if tgt is not None:
                    gemm_nt(Wmr.t().view(1, 1, Fd, Fd), dWf.transpose(-1, -2), out=tgt.view(M, 1, Fd, Cd), accumulate=True,
                            round_out=False)
                else:
                    dWv = gemm_nt(Wmr.t().view(1, 1, Fd, Fd), dWf.transpose(-1, -2), round_out=False).view(wv_shape)
        return da, dWv, dWm, None, None


def folded_value_bank(a, Wv, Wm, M, tag="small"):
    return _FoldedValueBank.apply(a, Wv, Wm, M, tag)


def attn_pv_gelu(P, v, M, bias, drop_p=0.0, seed=0):
    return _AttnPVGelu.apply(P, v, M, bias, drop_p, seed)


class _AttnPVGeluGroupLinear(torch.autograd.Function):
    """Y[b,m] = dropout(gelu(P[b,m] V'[b,:,m] + bm)) Wo[m]^T + bo[m]: _AttnPVGelu followed by _GroupLinear as ONE autograd
    node, so that backward can fuse gelu'(h) * dropout mask into the epilogue of the dG = dY Wo GEMM (SX_ACT_GELU_BWD)
    instead of writing dG, re-reading it with the pre-activation and writing dH in a separate pass."""

    @staticmethod
    def forward(ctx, P, v, M, bm, drop_p, seed, Wo, bo):
        B, _, U1, U2 = P.shape
        Fd = v.shape[-1] // M
        P = _rowpad(P)
        vv = v.view(B, U2, M, Fd).permute(0, 2, 3, 1)
        G = torch.empty((B, M, U1, Fd), device=P.device, dtype=torch.float32)
        H = torch.empty_like(G)
        gemm_nt(P, vv, out=G, bias=bm, gelu=True, preact=H, drop_p=drop_p, seed=seed)
        Wr = round_tf32(Wo).reshape(M, Fd, Fd)
        Y = torch.empty_like(G)
        gemm_nt(G, Wr.unsqueeze(0), out=Y, bias=bo.reshape(1, M, Fd), round_out=False)
        ctx.save_for_backward(P, v, H, G, Wr)
        ctx.meta = (M, Fd, drop_p, bm is not None, Wo.shape)
        ctx.seed = seed
        ctx.leaves = (bm, Wo, bo)
        return Y

    @staticmethod
    def backward(ctx, dY):
        P, v, H, G, Wr = ctx.saved_tensors
        M, Fd, drop_p, has_bm, wshape = ctx.meta
        bm, Wo, bo = ctx.leaves
        B, _, U1, U2 = P.shape
        dY = dY.contiguous()
        dP = dv = dbm = dW = dbo = None
        # dH = mask * (dY Wo) * gelu'(H), TF32-rounded for the two GEMMs that consume it
        dH = torch.empty_like(H)
        # ... and the column sums of dH (= the gradient of MMSharedMid's bias) are accumulated by the same epilogue
        dbm_buf = None
        if has_bm and ctx.needs_input_grad[3]:
            tgt = _grad_target(bm)
            dbm_buf = tgt if tgt is not None else _zeros((Fd,), dY.device)
            dbm = None if tgt is not None else dbm_buf
        gemm_nt(dY, Wr.transpose(-1, -2).unsqueeze(0), out=dH, gelu_bwd=H, drop_p=drop_p, seed=ctx.seed, colsum=dbm_buf)
        if ctx.needs_input_grad[6]:
            tgt = _grad_target(Wo)
            if tgt is not None:
                gemm_nt(dY.transpose(-1, -2), G.transpose(-1, -2), out=tgt.view(1, M, Fd, Fd), reduce_z1=True,
                        accumulate=True, round_out=False)
            else:
                dW = gemm_nt(dY.transpose(-1, -2), G.transpose(-1, -2), reduce_z1=True, round_out=False).view(wshape)
        if ctx.needs_input_grad[7]:
            tgt = _grad_target(bo)
            dbo_buf = tgt if tgt is not None else _zeros((M * Fd,), G.device)
            L.call("sx_colsum_batched", dY.data_ptr(), B, M * U1 * Fd, M, U1 * Fd, U1, Fd, Fd, dbo_buf.data_ptr(), *_part_args(dY.device), _stream())
            dbo = None if tgt is not None else dbo_buf
        if ctx.needs_input_grad[0]:
            dP = _rowpad_empty((B, M, U1, U2), P.device)
            gemm_nt(dH, v.view(B, U2, M, Fd).permute(0, 2, 1, 3), out=dP, round_out=False)
        if ctx.needs_input_grad[1]:
            dv = torch.empty_like(v)
            gemm_nt(P.transpose(-1, -2), dH.transpose(-1, -2), out=dv.view(B, U2, M, Fd).permute(0, 2, 1, 3),
                    round_out=False)
        return dP, dv, None, dbm, None, None, dW, dbo


def attn_pv_gelu_group_linear(P, v, M, bm, drop_p, seed, Wo, bo):
    return _AttnPVGeluGroupLinear.apply(P, v, M, bm, drop_p, seed, Wo, bo)


# Fused squeeze-out attention (opt-out: set_attn_fusion(False)): scores + clamp + softmax + attention dropout run in
# csrc/sx_attn.cu (S never reaches HBM in inference; in training the raw scores are kept for the backward, which
# recomputes P in the epilogue of the dP GEMM instead of running a softmax-backward pass over P and dP).
_ATTN_FUSION = True


def set_attn_fusion(on: bool):
    global _ATTN_FUSION
    _ATTN_FUSION = bool(on)


def attn_fusion_enabled() -> bool:
    return _ATTN_FUSION and _PRECISION == "tf32"          # the 3-pass validation mode keeps the unfused fp32-grade products


class _SqueezeOutFused(torch.autograd.Function):
    """Y[b,m] = dropout(gelu(P[b,m] V'[b,:,m] + bm)) Wo[m]^T + bo[m]  with  P = dropout(softmax(min(Q K^T/sqrt(d), clip)))
    — CrossAttFeatTrans.forward (segtran_shared.py:566-605) + ExpandedFeatTrans up to MMPrivateOutput's Linear
    (:447, :243-245, :267) as ONE autograd node:
      forward : sx_attn_probs_fwd (wgmma scores -> in-register softmax -> P)  ->  P.V' GEMM (bias/GELU/dropout epilogue)
                -> grouped output Linear;
      backward: dH GEMM (GELU'/dropout epilogue + bias-gradient column sums) -> dP GEMM -> sx_softmax_bwd on the saved raw
                scores (P recomputed from S and the row log-sum-exp, the row term sum_a P_a dP_a taken from the SAME dP values
                it is subtracted from) -> dV', dQ, dK, dWo, dbo products.
    A flash-attention style backward (row term from sum_f dU_f U_f in the dH epilogue, softmax backward in the dP GEMM
    epilogue) was built and measured: its row term carries independent TF32 rounding, which the softmax Jacobian amplifies
    (input-gradient error 1.3e-2 at cfg 1 / cfg 4 against 6e-4 for this form), so it is not used."""

    @staticmethod
    def forward(ctx, q, k, vp, M, clip, att_p, att_seed, bm, hid_p, hid_seed, Wo, bo, diag, table=None, pb_geom=None):
        B, U2 = k.shape[0], k.shape[1]
        U1 = q.shape[1]
        Fd = vp.shape[-1] // M
        q = q.contiguous()
        k = k.contiguous()
        need_bwd = any(ctx.needs_input_grad)
        pb = PosBias(table, pb_geom[0], pb_geom[1], pb_geom[2]) if table is not None else None
        P, S, lse, _rowmax, stat = attn_probs_fused(q, k, M, clip, att_p, att_seed, diag, need_scores=need_bwd, posbias=pb)
        vv = vp.view(B, U2, M, Fd).permute(0, 2, 3, 1)
        G = torch.empty((B, M, U1, Fd), device=P.device, dtype=torch.float32)
        H = torch.empty_like(G)
        gemm_nt(P, vv, out=G, bias=bm, gelu=True, preact=H, drop_p=hid_p, seed=hid_seed)
        Wr = round_tf32(Wo).reshape(M, Fd, Fd)
        Y = torch.empty_like(G)
        gemm_nt(G, Wr.unsqueeze(0), out=Y, bias=bo.reshape(1, M, Fd), round_out=False)
        ctx.save_for_backward(q, k, P, S, lse, stat, vp, H, G, Wr)
        ctx.meta = (M, Fd, float(clip), att_p, hid_p, bm is not None, Wo.shape)
        ctx.seeds = (att_seed, hid_seed)
        ctx.leaves = (bm, Wo, bo)
        ctx.pb = (table, pb_geom)
        return Y

    @staticmethod
    def backward(ctx, dY):
        q, k, P, S, lse, stat, vp, H, G, Wr = ctx.saved_tensors
        M, Fd, clip, att_p, hid_p, has_bm, wshape = ctx.meta
        att_seed, hid_seed = ctx.seeds
        bm, Wo, bo = ctx.leaves
        table, pb_geom = ctx.pb
        dT = None
        B, _, U1, U2 = P.shape
        Bq, d = q.shape[0], q.shape[-1] // M
        dY = dY.contiguous()
        dq = dk = dvp = dbm = dW = dbo = None
        # dH = mask * (dY Wo) * gelu'(H); the same epilogue accumulates the column sums of dH (MMSharedMid's bias gradient)
        dH = torch.empty_like(H)
        dbm_buf = None
        if has_bm and ctx.needs_input_grad[7]:
            tgt = _grad_target(bm)
            dbm_buf = tgt if tgt is not None else _zeros((Fd,), dY.device)
            dbm = None if tgt is not None else dbm_buf
        gemm_nt(dY, Wr.transpose(-1, -2).unsqueeze(0), out=dH, gelu_bwd=H, drop_p=hid_p, seed=hid_seed, colsum=dbm_buf)
        if ctx.needs_input_grad[10]:
            tgt = _grad_target(Wo)
            if tgt is not None:
                gemm_nt(dY.transpose(-1, -2), G.transpose(-1, -2), out=tgt.view(1, M, Fd, Fd), reduce_z1=True,
                        accumulate=True, round_out=False)
            else:
                dW = gemm_nt(dY.transpose(-1, -2), G.transpose(-1, -2), reduce_z1=True, round_out=False).view(wshape)
        if ctx.needs_input_grad[11]:
            tgt = _grad_target(bo)
            dbo_buf = tgt if tgt is not None else _zeros((M * Fd,), G.device)
            L.call("sx_colsum_batched", dY.data_ptr(), B, M * U1 * Fd, M, U1 * Fd, U1, Fd, Fd, dbo_buf.data_ptr(), *_part_args(dY.device), _stream())
            dbo = None if tgt is not None else dbo_buf
        if ctx.needs_input_grad[2]:
            dvp = torch.empty_like(vp)
            gemm_nt(P.transpose(-1, -2), dH.transpose(-1, -2), out=dvp.view(B, U2, M, Fd).permute(0, 2, 1, 3),
                    round_out=False)
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1] or (table is not None and ctx.needs_input_grad[13]):
            dP = torch.empty_strided(P.size(), P.stride(), device=P.device, dtype=torch.float32)
            gemm_nt(dH, vp.view(B, U2, M, Fd).permute(0, 2, 1, 3), out=dP, round_out=False)
            dS = torch.empty_strided(P.size(), P.stride(), device=P.device, dtype=torch.float32)
            ld = P.stride(-2)
            if table is not None:
                dT = softmax_posbias_backward(dP, ld, S, ld, lse, B * M * U1, U2, stat[2:], clip, att_p, att_seed, ld, dS,
                                              ld, table, pb_geom, ctx.needs_input_grad[13])
            else:
                L.call("sx_softmax_bwd", dP.data_ptr(), ld, S.data_ptr(), ld, lse.data_ptr(), B * M * U1, U2,
                       stat[2:].data_ptr(), clip, att_p, *_seed_args(att_seed), ld, dS.data_ptr(), L.SX_F32, ld, _rt(), _stream())
            scale = 1.0 / math.sqrt(d)
            if ctx.needs_input_grad[0]:
                bcast = Bq == 1 and B > 1
                dq = _zeros_like(q) if bcast else torch.empty_like(q)
                gemm_nt(dS, k.view(B, U2, M, d).permute(0, 2, 3, 1), out=dq.view(Bq, U1, M, d).permute(0, 2, 1, 3),
                        alpha=scale, round_out=False, reduce_z1=bcast, split_k=1)
            if ctx.needs_input_grad[1]:
                dk = torch.empty_like(k)
                gemm_nt(dS.transpose(-1, -2), q.view(Bq, U1, M, d).permute(0, 2, 3, 1),
                        out=dk.view(B, U2, M, d).permute(0, 2, 1, 3), alpha=scale, round_out=False)
        return dq, dk, dvp, None, None, None, None, dbm, None, None, dW, dbo, None, dT, None


def _pb_args(posbias):
    if posbias is None:
        return None, None
    return _posbias_table(posbias), (posbias.R, posbias.grid, posbias.w)


def squeeze_out_fused(q, k, vp, M, clip, att_p, att_seed, bm, hid_p, hid_seed, Wo, bo, diag, posbias=None):
    """posbias (PosBias): sliding-window positional bias inside the softmax; its table receives a gradient."""
    return _SqueezeOutFused.apply(q, k, vp, M, clip, att_p, att_seed, bm, hid_p, hid_seed, Wo, bo, diag, *_pb_args(posbias))


class _LayerNorm(torch.autograd.Function):
    """nn.LayerNorm(C, eps=1e-12, affine) over the last dim (first_norm_layer, segtran_shared.py:456)."""

    @staticmethod
    def forward(ctx, x, g, b, rnd, rnd_bwd):
        ctx.rnd_bwd = rnd_bwd
        x = x.contiguous()
        Cd = x.shape[-1]
        R = x.numel() // Cd
        y = torch.empty_like(x)
        stats = torch.empty((R, 2), device=x.device, dtype=torch.float32)
        L.call("sx_layernorm_fwd", x.data_ptr(), R, Cd, g.data_ptr(), b.data_ptr(), y.data_ptr(), L.SX_F32, rnd,
               stats.data_ptr(), _stream())
        ctx.save_for_backward(x, g, stats)
        ctx.leaves = (g, b)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g, stats = ctx.saved_tensors
        dy = dy.contiguous()
        Cd = x.shape[-1]
        R = x.numel() // Cd
        dx = torch.empty_like(x)
        dgb, dg = _sink_or_zeros(ctx.leaves[0])
        dbb, db = _sink_or_zeros(ctx.leaves[1])
        L.call("sx_layernorm_bwd", dy.data_ptr(), x.data_ptr(), R, Cd, g.data_ptr(), stats.data_ptr(), dx.data_ptr(),
               L.SX_F32, ctx.rnd_bwd, dgb.data_ptr(), dbb.data_ptr(), *_part_args(dy.device), _stream())
        return dx, dg, db, None, None


class _GroupLinear(torch.autograd.Function):
    """Y[b,m] = G[b,m] Wo[m]^T + bo[m] — MMPrivateOutput's grouped 1x1 Conv1d (segtran_shared.py:267)."""

    @staticmethod
    def forward(ctx, G, Wo, bo):
        B, M, N, Fd = G.shape
        Wr = round_tf32(Wo).reshape(M, Fd, Fd)
        Y = torch.empty_like(G)
        gemm_nt(G, Wr.unsqueeze(0), out=Y, bias=bo.reshape(1, M, Fd), round_out=False)
        ctx.save_for_backward(G, Wr)
        ctx.wshape = Wo.shape
        ctx.leaves = (Wo, bo)
        return Y

    @staticmethod
    def backward(ctx, dY):
        G, Wr = ctx.saved_tensors
        B, M, N, Fd = G.shape
        dY = dY.contiguous()
        dG = dW = db = None
        if ctx.needs_input_grad[0]:
            dG = gemm_nt(dY, Wr.transpose(-1, -2).unsqueeze(0), round_out=False)
        Wo, bo = ctx.leaves
        if ctx.needs_input_grad[1]:
            tgt = _grad_target(Wo)
            if tgt is not None:
                gemm_nt(dY.transpose(-1, -2), G.transpose(-1, -2), out=tgt.view(1, M, Fd, Fd), reduce_z1=True,
                        accumulate=True, round_out=False)
            else:
                dW = gemm_nt(dY.transpose(-1, -2), G.transpose(-1, -2), reduce_z1=True, round_out=False)
                dW = dW.view(ctx.wshape)
        if ctx.needs_input_grad[2]:
            tgt = _grad_target(bo)
            db = tgt if tgt is not None else _zeros((M * Fd,), G.device)
            L.call("sx_colsum_batched", dY.data_ptr(), B, M * N * Fd, M, N * Fd, N, Fd, Fd, db.data_ptr(), *_part_args(dY.device), _stream())
            if tgt is not None:
                db = None
        return dG, dW, db


class _LnSoftAggr(torch.autograd.Function):
    """out = sum_m softmax_m(Yn_m.ws+bs) Yn_m, Yn = LN(dropout(Y))   (segtran_shared.py:273-274, :318-325)."""

    @staticmethod
    def forward(ctx, Y, g, b, ws, bs, drop_p, seed):
        Y = Y.contiguous()
        B, M, N, Fd = Y.shape
        out = torch.empty((B, N, Fd), device=Y.device, dtype=torch.float32)
        stats = torch.empty((B, M, N, 2), device=Y.device, dtype=torch.float32)
        wts = torch.empty((B, M, N), device=Y.device, dtype=torch.float32)
        L.call("sx_ln_softaggr_fwd", Y.data_ptr(), B, M, N, Fd, g.data_ptr(), b.data_ptr(), ws.data_ptr(),
               bs.data_ptr(), drop_p, *_seed_args(seed), out.data_ptr(), stats.data_ptr(), wts.data_ptr(), _stream())
        ctx.save_for_backward(Y, g, b, ws, stats, wts)
        ctx.meta = (drop_p, seed, bs.shape, ws.shape)
        ctx.leaves = (g, b, ws, bs)
        return out

    @staticmethod
    def backward(ctx, dout):
        Y, g, b, ws, stats, wts = ctx.saved_tensors
        drop_p, seed, bs_shape, ws_shape = ctx.meta
        B, M, N, Fd = Y.shape
        dout = dout.contiguous()
        dY = torch.empty_like(Y)
        dgb, dg = _sink_or_zeros(ctx.leaves[0])
        dbb, db = _sink_or_zeros(ctx.leaves[1])
        dwsb, dws = _sink_or_zeros(ctx.leaves[2])
        dbsb, dbs = _sink_or_zeros(ctx.leaves[3])
        scratch = torch.empty(B * M * N, device=Y.device, dtype=torch.float32)
        L.call("sx_ln_softaggr_bwd", dout.data_ptr(), Y.data_ptr(), B, M, N, Fd, g.data_ptr(), b.data_ptr(),
               ws.data_ptr(), drop_p, *_seed_args(seed), stats.data_ptr(), wts.data_ptr(), dY.data_ptr(), L.SX_F32, _rt(), dgb.data_ptr(),
               dbb.data_ptr(), dwsb.data_ptr(), dbsb.data_ptr(), scratch.data_ptr(), *_part_args(dout.device), _stream())
        return dY, dg, db, dws, dbs, None, None


class _SoftAggr(torch.autograd.Function):
    """out = sum_m softmax_m(x_m . ws + bs) x_m  — LearnedSoftAggregate (segtran_shared.py:318-325) without a LayerNorm in
    front: the no-FFN branch of ExpandedFeatTrans (:453) with M modes, i.e. the Polyformer layer.  x [B,M,N,F] -> [B,N,F]."""

    @staticmethod
    def forward(ctx, x, ws, bs):
        x = x.contiguous()
        B, M, N, Fd = x.shape
        wsc, bsc = ws.contiguous().view(-1), bs.contiguous().view(-1)
        out = torch.empty((B, N, Fd), device=x.device, dtype=torch.float32)
        wts = torch.empty((B, M, N), device=x.device, dtype=torch.float32)
        L.call("sx_softaggr_fwd", x.data_ptr(), B, M, N, Fd, wsc.data_ptr(), bsc.data_ptr(), out.data_ptr(), wts.data_ptr(),
               _stream())
        ctx.save_for_backward(x, wsc, wts)
        ctx.shapes = (ws.shape, bs.shape)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, wsc, wts = ctx.saved_tensors
        B, M, N, Fd = x.shape
        dout = dout.contiguous()
        dx = torch.empty_like(x)
        dscore = torch.empty((B, M, N), device=x.device, dtype=torch.float32)
        L.call("sx_softaggr_bwd", dout.data_ptr(), x.data_ptr(), B, M, N, Fd, wsc.data_ptr(), wts.data_ptr(), dx.data_ptr(),
               dscore.data_ptr(), _stream())
        R = B * M * N
        dws = _sgemm(dscore, x, 1, Fd, R, (1, 1), (Fd, 1))[0].view(ctx.shapes[0])         # sum_r dscore[r] x[r,:]
        dbs = _zeros((1,), x.device)
        L.call("sx_rowsum", dscore.data_ptr(), 1, R, R, 1, dbs.data_ptr(), *_part_args(dscore.device), _stream())
        return dx, dws, dbs.view(ctx.shapes[1])


def soft_aggregate(x, ws, bs):
    return _SoftAggr.apply(x, ws, bs)


class _PosCode(torch.autograd.Function):
    """LearnedSinuPosEmbedder (segtran_shared.py:989-998) on pos/pos.max() (:1231): [R,pd] -> [R,C0]."""

    @staticmethod
    def forward(ctx, pos2d, W, b, normalize):
        pos2d = pos2d.contiguous().float()
        R, pd = pos2d.shape
        C0 = W.shape[0]
        if normalize:
            pmax = torch.empty(1, device=pos2d.device, dtype=torch.float32)
            L.call("sx_reduce_max", pos2d.data_ptr(), pos2d.numel(), pmax.data_ptr(), _stream())
        else:
            pmax = torch.ones(1, device=pos2d.device, dtype=torch.float32)
        pe = torch.empty((R, C0), device=pos2d.device, dtype=torch.float32)
        Wc, bc = W.contiguous(), b.contiguous()
        L.call("sx_pos_lsinu_fwd", pos2d.data_ptr(), pmax.data_ptr(), R, pd, Wc.data_ptr(), bc.data_ptr(), C0,
               pe.data_ptr(), _stream())
        ctx.save_for_backward(pos2d, pmax, Wc, bc)
        ctx.leaves = (W, b)
        return pe

    @staticmethod
    def backward(ctx, dpe):
        pos2d, pmax, W, b = ctx.saved_tensors
        R, pd = pos2d.shape
        C0 = W.shape[0]
        dpe = dpe.contiguous()
        scratch = torch.empty_like(dpe)
        dWb, dW = _sink_or_zeros(ctx.leaves[0], like=W)
        dbb, db = _sink_or_zeros(ctx.leaves[1], like=b)
        L.call("sx_pos_lsinu_bwd", pos2d.data_ptr(), pmax.data_ptr(), R, pd, W.data_ptr(), b.data_ptr(), C0,
               dpe.data_ptr(), scratch.data_ptr(), dWb.data_ptr(), dbb.data_ptr(), *_part_args(pos2d.device), _stream())
        return None, dW, db, None


class _Prologue(torch.autograd.Function):
    """h = mask * dropout(LN(LN_{g,b}(x) + posw * pe[:, :C]))   (segtran_shared.py:916, :930-934, :944-946);
    pe None (no positional code, :940): h = mask * dropout(LN_{g,b}(x))."""

    @staticmethod
    def forward(ctx, x, g, b, pe, posw, mask, drop_p, seed):
        x = x.contiguous()
        B, N, Cd = x.shape
        if pe is not None:
            pe = pe.contiguous()                   # [N, C0] shared by the batch, or [B, N, C0]
        C0 = pe.shape[-1] if pe is not None else 0
        pe_bstride = 0 if pe is None or pe.dim() == 2 else N * C0
        h = torch.empty_like(x)
        stats = torch.empty((B * N, 4), device=x.device, dtype=torch.float32)
        L.call("sx_prologue_fwd", x.data_ptr(), B, N, Cd, g.data_ptr(), b.data_ptr(), _ptr(pe), C0, pe_bstride,
               posw, _ptr(mask), drop_p, *_seed_args(seed), h.data_ptr(), L.SX_F32, _rt(), stats.data_ptr(), _stream())
        ctx.save_for_backward(x, g, b, pe, mask, stats)
        ctx.meta = (posw, drop_p, seed, pe_bstride)
        ctx.leaves = (g, b)
        return h

    @staticmethod
    def backward(ctx, dh):
        x, g, b, pe, mask, stats = ctx.saved_tensors
        posw, drop_p, seed, pe_bstride = ctx.meta
        B, N, Cd = x.shape
        C0 = pe.shape[-1] if pe is not None else 0
        dh = dh.contiguous()
        dx = torch.empty_like(x)
        dgb, dg = _sink_or_zeros(ctx.leaves[0])
        dbb, db = _sink_or_zeros(ctx.leaves[1])
        dpe = _zeros_like(pe) if pe is not None and ctx.needs_input_grad[3] else None
        scratch = torch.empty_like(x) if pe is not None else None
        L.call("sx_prologue_bwd", dh.data_ptr(), x.data_ptr(), B, N, Cd, g.data_ptr(), b.data_ptr(), _ptr(pe), C0,
               pe_bstride, posw, _ptr(mask), drop_p, *_seed_args(seed), stats.data_ptr(), dx.data_ptr(), dgb.data_ptr(), dbb.data_ptr(),
               _ptr(dpe), _ptr(scratch), *_part_args(dh.device), _stream())
        if pe is None:
            L.launch_count -= 1             # without a code: row kernel + part_reduce, one fewer than _LAUNCHES counts
        return dx, dg, db, dpe, None, None, None, None


class _Transpose(torch.autograd.Function):
    """[Z,R,C] -> [Z,C,R]: token flatten / scatter (segtran3d.py:328-330, :478-480)."""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        Z, R, Cd = x.shape
        y = torch.empty((Z, Cd, R), device=x.device, dtype=torch.float32)
        L.call("sx_transpose", x.data_ptr(), Z, R, Cd, y.data_ptr(), _stream())
        return y

    @staticmethod
    def backward(ctx, dy):
        return _Transpose.apply(dy)


class _Dot(torch.autograd.Function):
    """loss = sum(x * w) for a fixed weight tensor w (a linear stand-in for the training loss in benchmarks)."""

    @staticmethod
    def forward(ctx, x, w):
        x = x.contiguous()
        out = _zeros((1,), x.device)
        L.call("sx_dot", x.data_ptr(), w.data_ptr(), x.numel(), out.data_ptr(), _stream())
        ctx.save_for_backward(w)
        ctx.shape = x.shape
        return out

    @staticmethod
    def backward(ctx, g):
        (w,) = ctx.saved_tensors
        dx = torch.empty_like(w)
        g = g.contiguous()
        L.call("sx_scale", w.data_ptr(), w.numel(), g.data_ptr(), 1.0, dx.data_ptr(), _stream())
        return dx.view(ctx.shape), None


def dot(x, w):
    return _Dot.apply(x, w.contiguous())


def attn_scores(q, k, M, amax=None, row_bias=None, tag="big", alpha=None):
    """alpha: score scale (default 1/sqrt(d) of the per-mode width)."""
    return _AttnScores.apply(q, k, M, amax, row_bias, tag, alpha)


def softmax(S, amax=None, clip=500.0, drop_p=0.0, seed=0, diag=None):
    """diag: optional device float[2] updated in place: [0] = max(diag[0], *amax), [1] += (*amax > clip)."""
    return _Softmax.apply(S, amax, clip, drop_p, seed, diag)


def softmax_posbias(S, posbias, amax=None, clip=500.0, drop_p=0.0, seed=0, diag=None):
    """softmax() with the sliding-window positional bias added after the clamp; S [B,M,N,N] with N = posbias.num_tokens."""
    if S.shape[-1] != posbias.num_tokens or S.shape[-2] != posbias.num_tokens:
        raise L.SxError("softmax_posbias: scores %s do not match the %s bias grid" % (tuple(S.shape), posbias.grid))
    table, geom = _pb_args(posbias)
    return _SoftmaxPosBias.apply(S, amax, clip, drop_p, seed, diag, table, geom)


def attn_pv(P, v, M, tag="big", round_out=True):
    return _AttnPV.apply(P, v, M, tag, round_out)


def layer_norm(x, g, b, consumer_tag=None, producer_tag=None):
    """consumer_tag / producer_tag: precision class of the contractions that consume y / that produced x (they decide
    whether y, respectively dx, is TF32-rounded here)."""
    return _LayerNorm.apply(x, g, b, _rt() if consumer_tag is None else rt_for(consumer_tag),
                            _rt() if producer_tag is None else rt_for(producer_tag))


def group_linear(G, Wo, bo):
    return _GroupLinear.apply(G, Wo, bo)


def ln_softaggr(Y, g, b, ws, bs, drop_p=0.0, seed=0):
    return _LnSoftAggr.apply(Y, g, b, ws, bs, drop_p, seed)


def pos_code(pos2d, W, b, normalize=True):
    """normalize: divide the positions by their global maximum first (SegtranPosEncoder.forward, :1231)."""
    return _PosCode.apply(pos2d, W, b, bool(normalize))


def prologue(x, g, b, pe, posw, mask, drop_p=0.0, seed=0):
    return _Prologue.apply(x, g, b, pe, posw, mask, drop_p, seed)


def transpose(x):
    return _Transpose.apply(x)


# ------------------------------------------------------------------------------------------------
# collapsed segmentation head (csrc/sx_head.cu)
# ------------------------------------------------------------------------------------------------
def _resize_axis(x: torch.Tensor, axis: int, Lout: int, accumulate_into: Optional[torch.Tensor] = None):
    shp = list(x.shape)
    Lin = shp[axis]
    outer = 1
    for s in shp[:axis]:
        outer *= s
    inner = 1
    for s in shp[axis + 1:]:
        inner *= s
    shp[axis] = Lout
    if accumulate_into is not None:
        y = accumulate_into
        acc = 1
    else:
        y = torch.empty(shp, device=x.device, dtype=torch.float32)
        acc = 0
    L.call("sx_resize_axis_fwd", x.data_ptr(), outer, Lin, Lout, inner, y.data_ptr(), acc, _stream())
    return y


def _resize_axis_adj(dy: torch.Tensor, axis: int, Lin: int):
    shp = list(dy.shape)
    Lout = shp[axis]
    outer = 1
    for s in shp[:axis]:
        outer *= s
    inner = 1
    for s in shp[axis + 1:]:
        inner *= s
    shp[axis] = Lin
    dx = torch.empty(shp, device=dy.device, dtype=torch.float32)
    L.call("sx_resize_axis_bwd", dy.data_ptr(), outer, Lin, Lout, inner, dx.data_ptr(), _stream())
    return dx


class _Resize(torch.autograd.Function):
    """F.interpolate(x, size, mode='bi/trilinear', align_corners=False) on the trailing dims, one pass per axis."""

    @staticmethod
    def forward(ctx, x, size):
        x = x.contiguous()
        nd = len(size)
        ctx.in_sizes = tuple(x.shape[-nd:])
        y = x
        for i, s in enumerate(size):
            ax = x.dim() - nd + i
            if y.shape[ax] != s:
                y = _resize_axis(y, ax, s)
        ctx.size = tuple(size)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        nd = len(ctx.size)
        for i in reversed(range(nd)):
            ax = dy.dim() - nd + i
            if ctx.in_sizes[i] != ctx.size[i]:
                dy = _resize_axis_adj(dy, ax, ctx.in_sizes[i])
        return dy, None


def resize_linear(x, size):
    return _Resize.apply(x, tuple(int(s) for s in size))


# ------------------------------------------------------------------------------------------------
# token-grid resampling (mince transformer, segtran_shared.py:45-66): csrc/sx_resample.cu
# ------------------------------------------------------------------------------------------------
def _f32(v) -> float:
    return float(np.float32(v))


def down_ratio(scale) -> float:
    """Source cells per output cell of F.interpolate(scale_factor=1/scale): 1/scale_factor, rounded to fp32 as PyTorch's
    kernels do (so a 7-cell axis at scale 2 becomes 3 cells read at stride 2.0)."""
    return _f32(1.0 / (1.0 / float(scale)))


def size_ratio(lin, lout) -> float:
    """Source cells per output cell of F.interpolate(size=...): Lin/Lout in fp32."""
    return float(np.float32(lin) / np.float32(lout))


def _resample_grid(lin, lout, ratios) -> L.sx_resample_grid:
    if len(lin) not in (1, 2, 3) or len(lout) != len(lin) or len(ratios) != len(lin):
        raise L.SxError("resize_tokens: 1-D to 3-D grids expected (got %s -> %s)" % (tuple(lin), tuple(lout)))
    pad = 3 - len(lin)
    g = L.sx_resample_grid()
    for a in range(3):
        u = a - pad
        g.lin[a], g.lout[a], g.ratio[a] = (int(lin[u]), int(lout[u]), float(ratios[u])) if u >= 0 else (1, 1, 1.0)
    return g


def _cells(grid) -> int:
    n = 1
    for v in grid:
        n *= int(v)
    return n


def _tok_layout(t: torch.Tensor, G: int):
    """(batch, group, row) strides of a contiguous token-major [B, N, G*D] tensor, and D."""
    B, N, C = t.shape
    return (N * C, C // G, C), C // G


def _mode_layout(t: torch.Tensor):
    """(batch, group, row) strides of a contiguous mode-major [B, G, N, W] tensor."""
    B, G, N, W = t.shape
    return (G * N * W, N * W, W)


def _resize_fwd(x, xs, y, ys, B, G, w, w_pad, grid, rnd):
    L.call("sx_resize_tokens_fwd", x, *xs, y, *ys, B, G, w, w_pad, C.byref(grid), rnd, _stream())


def _resize_bwd(dy, ys, dx, xs, B, G, w, w_pad, grid, acc):
    L.call("sx_resize_tokens_bwd", dy, *ys, dx, *xs, B, G, w, w_pad, C.byref(grid), acc, _stream())


class _ResizeTokensDown(torch.autograd.Function):
    """Per window s: y_s [B, N_s, G*w_pad_s] = resample of the channel window [c0_s, c1_s) of every group of the token-major
    x [B, N, G*D] from `grid` to grids_out[s] (ratios[s]); columns [w_s, w_pad_s) of each group are zeros.
    Backward: the windows of dx are written one by one (no zero-fill when they tile [0, D))."""

    @staticmethod
    def forward(ctx, x, G, grid, grids_out, ratios, windows, w_pads, round_out):
        _req_cuda(x)
        x = x.contiguous()
        B = x.shape[0]
        xs, D = _tok_layout(x, G)
        outs = []
        for g_out, r, (c0, c1), wp in zip(grids_out, ratios, windows, w_pads):
            y = torch.empty((B, _cells(g_out), G * wp), device=x.device, dtype=torch.float32)
            _resize_fwd(x.data_ptr() + 4 * c0, xs, y.data_ptr(), _tok_layout(y, G)[0], B, G, c1 - c0, wp,
                        _resample_grid(grid, g_out, r), _rt() if round_out else 0)
            outs.append(y)
        ctx.meta = (x.shape, G, tuple(grid), [tuple(g) for g in grids_out], ratios, windows, w_pads)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *dys):
        shape, G, grid, grids_out, ratios, windows, w_pads = ctx.meta
        B, N, Cx = shape
        D = Cx // G
        tiled = sorted(windows)[0][0] == 0 and sorted(windows)[-1][1] == D and \
            all(a[1] == b[0] for a, b in zip(sorted(windows), sorted(windows)[1:]))
        dx = (torch.empty if tiled else torch.zeros)(shape, device=dys[0].device, dtype=torch.float32)
        xs = (N * Cx, D, Cx)
        for dy, g_out, r, (c0, c1), wp in zip(dys, grids_out, ratios, windows, w_pads):
            dy = dy.contiguous()
            _resize_bwd(dy.data_ptr(), _tok_layout(dy, G)[0], dx.data_ptr() + 4 * c0, xs, B, G, c1 - c0, c1 - c0,
                        _resample_grid(grid, g_out, r), 0)
        return dx, None, None, None, None, None, None, None


def resize_tokens(x, G, grid, grids_out, ratios, windows, w_pads=None, round_out=True):
    """Linear / bilinear / trilinear resampling (align_corners=False) of channel windows of token-major rows.
    x [B, N, G*D] (N = cells of the row-major `grid`); windows [(c0, c1), ...] of each group's D channels; grids_out and
    ratios (per axis, see down_ratio / size_ratio) per window.  -> tuple of [B, N_s, G*w_pad_s] (w_pad_s defaults to
    c1-c0 rounded up to 4; padding columns are zero), TF32-rounded for a GEMM consumer unless round_out=False."""
    if w_pads is None:      # 16-byte GEMM operand strides: 4 fp32 columns, 8 when the products run on bf16 copies
        w_pads = [((c1 - c0 + 7) // 8 * 8) if _PRECISION == "bf16" else _pad4(c1 - c0) for c0, c1 in windows]
    return _ResizeTokensDown.apply(x, int(G), tuple(int(v) for v in grid), [tuple(int(v) for v in g) for g in grids_out],
                                   [tuple(float(r) for r in rs) for rs in ratios], [(int(a), int(b)) for a, b in windows],
                                   [int(w) for w in w_pads], bool(round_out))


class _ResizeTokensUpInto(torch.autograd.Function):
    """U [B, G, N, F] with its channel window [c0_s, c1_s) = resample of us[s][..., :c1_s-c0_s] ([B, G, N_s, W_s],
    mode-major) from grids_in[s] to `grid` (ratios[s]); the windows tile [0, F), so every element of U is written once.
    Backward: each dus[s] reads its window of dU (padding columns [c1_s-c0_s, W_s) zero)."""

    @staticmethod
    def forward(ctx, grid, grids_in, ratios, windows, Fd, round_out, *us):
        B, G = us[0].shape[0], us[0].shape[1]
        N = _cells(grid)
        U = torch.empty((B, G, N, Fd), device=us[0].device, dtype=torch.float32)
        Us = _mode_layout(U)
        for u, g_in, r, (c0, c1) in zip(us, grids_in, ratios, windows):
            u = u.contiguous()
            _resize_fwd(u.data_ptr(), _mode_layout(u), U.data_ptr() + 4 * c0, Us, B, G, c1 - c0, c1 - c0,
                        _resample_grid(g_in, grid, r), _rt() if round_out else 0)
        ctx.meta = (tuple(grid), grids_in, ratios, windows, [tuple(u.shape) for u in us])
        return U

    @staticmethod
    def backward(ctx, dU):
        grid, grids_in, ratios, windows, ushapes = ctx.meta
        dU = dU.contiguous()
        B, G = dU.shape[0], dU.shape[1]
        dUs = _mode_layout(dU)
        dus = []
        for g_in, r, (c0, c1), ush in zip(grids_in, ratios, windows, ushapes):
            du = torch.empty(ush, device=dU.device, dtype=torch.float32)
            _resize_bwd(dU.data_ptr() + 4 * c0, dUs, du.data_ptr(), _mode_layout(du), B, G, c1 - c0, ush[-1],
                        _resample_grid(g_in, grid, r), 0)
            dus.append(du)
        return (None, None, None, None, None, None) + tuple(dus)


def resize_tokens_into(us, grid, grids_in, windows, Fd, round_out=True):
    """Upsample each us[s] [B, G, N_s, W_s] (mode-major, e.g. P_s.V_s) to the full `grid` with F.interpolate(size=grid)
    semantics, writing channel window windows[s] of ONE [B, G, N, Fd] tensor (the concatenation over the windows)."""
    ratios = [tuple(size_ratio(a, b) for a, b in zip(g_in, grid)) for g_in in grids_in]
    return _ResizeTokensUpInto.apply(tuple(int(v) for v in grid), [tuple(int(v) for v in g) for g in grids_in], ratios,
                                     [(int(a), int(b)) for a, b in windows], int(Fd), bool(round_out), *us)


class _AttnProbs(torch.autograd.Function):
    """P = dropout(softmax(clamp_if(alpha Q K^T) [+ w bias])) per mode as one node over the fused kernel
    (attn_probs_fused): backward = softmax backward on the saved raw scores (sx_softmax_bwd / softmax_posbias_backward,
    with the table gradient) -> dQ, dK products."""

    @staticmethod
    def forward(ctx, q, k, M, alpha, clip, drop_p, seed, diag, table, pb_geom):
        pb = PosBias(table, *pb_geom) if table is not None else None
        need_bwd = any(ctx.needs_input_grad)
        P, S, lse, _rowmax, stat = attn_probs_fused(q, k, M, clip, drop_p, seed, diag, need_scores=need_bwd, posbias=pb,
                                                    alpha=alpha)
        ctx.save_for_backward(q, k, S, lse, stat)
        ctx.meta = (M, alpha, clip, drop_p, P.stride(-2), pb_geom)
        ctx.seed = seed
        ctx.leaf = table
        return P

    @staticmethod
    def backward(ctx, dP):
        q, k, S, lse, stat = ctx.saved_tensors
        M, alpha, clip, drop_p, ldp, pb_geom = ctx.meta
        table = ctx.leaf
        B, _, U1, U2 = S.shape
        dP = _rowpad(dP)
        dS = _rowpad_empty(S.shape, S.device)
        dT = None
        if table is not None:
            dT = softmax_posbias_backward(dP, dP.stride(-2), S, S.stride(-2), lse, B * M * U1, U2, stat[2:], clip, drop_p,
                                          ctx.seed, ldp, dS, dS.stride(-2), table, pb_geom, ctx.needs_input_grad[8])
        else:
            L.call("sx_softmax_bwd", dP.data_ptr(), dP.stride(-2), S.data_ptr(), S.stride(-2), lse.data_ptr(), B * M * U1, U2,
                   stat[2:].data_ptr(), clip, drop_p, *_seed_args(ctx.seed), ldp, dS.data_ptr(), L.SX_F32, dS.stride(-2),
                   _rt(), _stream())
        dq, dk = _score_grads(dS, q, k, M, alpha, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return dq, dk, None, None, None, None, None, None, dT, None


def attn_probs(q, k, M, alpha, clip=500.0, drop_p=0.0, seed=0, diag=None, posbias=None):
    """Differentiable fused attention probabilities (see _AttnProbs); q, k [B, U, M*d] contiguous, TF32-rounded."""
    return _AttnProbs.apply(q.contiguous(), k.contiguous(), M, float(alpha), float(clip), drop_p, seed, diag,
                            *_pb_args(posbias))


def _sgemm(A, B, M, N, K, sa, sb, out=None, alpha=1.0, accumulate=False, Z=1, zs=(0, 0, 0)):
    """C[z](m,n) (+)= alpha sum_k A[z](m,k) B[z](k,n); sa=(sam,sak), sb=(sbk,sbn); out [Z,M,N] contiguous."""
    if out is None:
        out = torch.empty((Z, M, N), device=A.device, dtype=torch.float32)
    L.call("sx_sgemm_small", A.data_ptr(), B.data_ptr(), out.data_ptr(), M, N, K, sa[0], sa[1], sb[0], sb[1], N, 1, Z,
           zs[0], zs[1], M * N if zs[2] is None else zs[2], alpha, 1 if accumulate else 0, _stream())
    return out


class _HeadContract(torch.autograd.Function):
    """L[b,k,v] = sum_c (Wc Wb)[k,c] curr[b,c,v] + (Wc bb + bc)[k] + tvup[b,k,v]
    with curr [B,Cf,*sp], Wb [F,Cf] (bridge conv), bb [F], Wc [K,F] (class conv), bc [K].
    Collapsed form of conv_cls(conv_bridge(curr) + up) before interpolation (segtran3d.py:364-367, :488-490)."""

    @staticmethod
    def forward(ctx, curr, Wb, bb, Wc, bc, tvup):
        curr = curr.contiguous()
        B, Cf = curr.shape[:2]
        V = curr[0, 0].numel()
        K, Fd = Wc.shape
        Wb2 = Wb.reshape(Fd, Cf).contiguous() if Wb is not None else None
        Wc2 = Wc.contiguous()
        if Wb2 is not None:
            Wcb = _sgemm(Wc2, Wb2, K, Cf, Fd, (Fd, 1), (Cf, 1))[0]                      # [K,Cf]
            cc = bc.detach().clone().contiguous() if bc is not None else torch.zeros(K, device=curr.device)
            _sgemm(Wc2, bb.contiguous(), K, 1, Fd, (Fd, 1), (1, 1), out=cc.view(1, K, 1), accumulate=True)   # += Wc bb
        else:                                   # bridge conv is nn.Identity (segtran2d.py:177-180): Cf == F
            Wcb = Wc2
            cc = bc.contiguous() if bc is not None else torch.zeros(K, device=curr.device)
        Lo = tvup.contiguous().clone() if tvup is not None else torch.zeros((B, K, V), device=curr.device)
        L.call("sx_head_contract_fwd", curr.data_ptr(), Wcb.data_ptr(), cc.data_ptr(), B, Cf, V, K, Lo.data_ptr(), 1,
               _stream())
        ctx.save_for_backward(curr, Wb2, bb, Wc2, Wcb)
        ctx.meta = (Wb.shape if Wb is not None else None, tvup is not None, bc is not None)
        return Lo.view(B, K, *curr.shape[2:])

    @staticmethod
    def backward(ctx, dL):
        curr, Wb2, bb, Wc2, Wcb = ctx.saved_tensors
        wb_shape, has_tv, has_bc = ctx.meta
        B, Cf = curr.shape[:2]
        V = curr[0, 0].numel()
        K, Fd = Wc2.shape
        dL = dL.contiguous()
        dcurr = dWb = dbb = dWc = dbc = dtv = None
        if ctx.needs_input_grad[0]:
            dcurr = torch.empty_like(curr)
            L.call("sx_head_contract_bwd_data", dL.data_ptr(), Wcb.data_ptr(), B, Cf, V, K, dcurr.data_ptr(), _stream())
        # dWcb[k,c] = sum_{b,v} dL[b,k,v] curr[b,c,v]: a (K x Cf x B*V) product streamed once through the tensor
        # cores (TF32 operands, fp32 accumulation; HBM-bound on reading curr), reduced over the batch atomically
        need_w = any(ctx.needs_input_grad[1:5])
        if not need_w:
            return dcurr, None, None, None, None, (dL.view(B, K, V) if has_tv else None)
        if V % 4 == 0:
            dWcb = gemm_nt(dL.view(B, 1, K, V), curr.view(B, 1, Cf, V), reduce_z1=True, round_out=False).view(K, Cf)
        else:                                         # TMA needs 16-byte row pitches: CUDA-core reduction instead
            dWcb = _zeros((K, Cf), curr.device)
            L.call("sx_head_contract_bwd_weight", dL.data_ptr(), curr.data_ptr(), B, Cf, V, K, dWcb.data_ptr(), _stream())
        dcc = _zeros((K,), curr.device)               # d(const)[k] = sum_{b,v} dL
        L.call("sx_rowsum", dL.data_ptr(), B * K, V, V, K, dcc.data_ptr(), *_part_args(dL.device), _stream())
        if Wb2 is not None:
            # Wcb = Wc Wb ; cc = Wc bb + bc
            dWc = gemm_nt(dWcb, Wb2, round_out=False).view(1, K, Fd)                  # dWcb Wb^T   [K,F]
            _sgemm(dcc, bb.contiguous(), K, Fd, 1, (1, 1), (1, 1), out=dWc, accumulate=True)
            dWc = dWc[0]
            dWb = _sgemm(Wc2, dWcb, Fd, Cf, K, (1, Fd), (Cf, 1))[0].reshape(wb_shape)   # Wc^T dWcb  [F,Cf]
            dbb = _sgemm(Wc2, dcc, Fd, 1, K, (1, Fd), (1, 1))[0].reshape(Fd)           # Wc^T dcc
        else:
            dWc = dWcb
        if has_bc:
            dbc = dcc
        if has_tv:
            dtv = dL.view(B, K, V)
        return dcurr, dWb, dbb, dWc, dbc, dtv


class _TokenClassScores(torch.autograd.Function):
    """tvT[b,k,n] = sum_f Wc[k,f] vf[b,n,f] — class scores of the fused tokens, channels-first."""

    @staticmethod
    def forward(ctx, vf, Wc):
        vf = vf.contiguous()
        Wc = Wc.contiguous()
        B, N, Fd = vf.shape
        K = Wc.shape[0]
        out = torch.empty((B, K, N), device=vf.device, dtype=torch.float32)
        L.call("sx_token_scores", vf.data_ptr(), Wc.data_ptr(), B, N, Fd, K, out.data_ptr(), _stream())   # exact fp32
        ctx.save_for_backward(vf, Wc)
        return out

    @staticmethod
    def backward(ctx, dt):
        vf, Wc = ctx.saved_tensors
        B, N, Fd = vf.shape
        K = Wc.shape[0]
        dt = dt.contiguous()
        # dvf[b,n,f] = sum_k dt[b,k,n] Wc[k,f]      (K = num_classes: CUDA-core product, coalesced over f)
        if Fd % 4 == 0:
            dvf = torch.empty_like(vf)
            L.call("sx_token_scores_bwd", dt.data_ptr(), Wc.data_ptr(), B, N, Fd, K, dvf.data_ptr(), _stream())
        else:
            dvf = _sgemm(dt, Wc, N, Fd, K, (1, N), (Fd, 1), Z=B, zs=(K * N, 0, N * Fd))
        # dWc[k,f] = sum_{b,n} dt[b,k,n] vf[b,n,f]  (tensor cores, reduced over the batch)
        if N % 4 == 0:
            dWc = gemm_nt(dt.view(B, 1, K, N), vf.transpose(1, 2).unsqueeze(1), reduce_z1=True, round_out=False)
            dWc = dWc.view(K, Fd)
        else:
            dWc = _zeros((1, K, Fd), vf.device)
            for bi in range(B):
                _sgemm(dt[bi], vf[bi], K, Fd, N, (N, 1), (Fd, 1), out=dWc, accumulate=True)
            dWc = dWc[0]
        return dvf, dWc


# ------------------------------------------------------------------------------------------------
# FPN pyramid stage (SURVEY §8 f.1): curr <- GroupNorm(conv1x1(curr) + upsample(higher))   on channels-first tensors
# ------------------------------------------------------------------------------------------------
class _Conv1x1Add(torch.autograd.Function):
    """y[b] = W x[b] + bias (+ addend[b]) for channels-first x [B,Cin,V]: a 1x1(x1) convolution with the "add the
    upsampled coarser level" of an FPN stage in its epilogue (segtran3d.py:300-306, :348-354).  One GEMM: W is the K-major
    A operand broadcast over the batch, x[b] is read in place as an MN-major [V x Cin] operand."""

    @staticmethod
    def forward(ctx, x, W, b, addend):
        B, Cin, V = x.shape
        Cout = W.shape[0]
        xr = round_tf32(x)                                   # the level below comes from outside (backbone): round once
        Wr = round_tf32(W).reshape(Cout, Cin)
        y = torch.empty((B, 1, Cout, V), device=x.device, dtype=torch.float32)
        ad = None if addend is None else addend.contiguous().view(B, 1, Cout, V)
        gemm_nt(Wr.view(1, 1, Cout, Cin), xr.view(B, 1, Cin, V).transpose(-1, -2), out=y, bias=b, bias_mode=L.SX_BIAS_M,
                addend=ad, round_out=False)
        ctx.save_for_backward(xr, Wr)
        ctx.meta = (W.shape, b is not None, addend is not None)
        ctx.leaves = (W, b)
        return y.view(B, Cout, V)

    @staticmethod
    def backward(ctx, dy):
        xr, Wr = ctx.saved_tensors
        wshape, has_b, has_add = ctx.meta
        W, b = ctx.leaves
        B, Cin, V = xr.shape
        Cout = Wr.shape[0]
        dy = dy.contiguous()
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            dx = gemm_nt(Wr.t().view(1, 1, Cin, Cout), dy.view(B, 1, Cout, V).transpose(-1, -2), round_out=False)
            dx = dx.view(B, Cin, V)
        if ctx.needs_input_grad[1]:
            tgt = _grad_target(W)
            if tgt is not None:
                gemm_nt(dy.view(B, 1, Cout, V), xr.view(B, 1, Cin, V), out=tgt.view(1, 1, Cout, Cin), reduce_z1=True,
                        accumulate=True, round_out=False)
            else:
                dW = gemm_nt(dy.view(B, 1, Cout, V), xr.view(B, 1, Cin, V), reduce_z1=True, round_out=False).view(wshape)
        if has_b and ctx.needs_input_grad[2]:
            tgt = _grad_target(b)
            buf = tgt if tgt is not None else _zeros((Cout,), dy.device)
            L.call("sx_rowsum", dy.data_ptr(), B * Cout, V, V, Cout, buf.data_ptr(), *_part_args(dy.device), _stream())
            db = None if tgt is not None else buf
        return dx, dW, db, (dy if has_add else None)


class _GroupNorm(torch.autograd.Function):
    """nn.GroupNorm(G, C) on channels-first [B,C,V] (segtran3d.py:150, :174; eps 1e-5): one reduction pass + one apply pass."""

    @staticmethod
    def forward(ctx, x, gamma, beta, G, eps, round_out):
        x = x.contiguous()
        B, Cd, V = x.shape
        y = torch.empty_like(x)
        csum = torch.empty(B * Cd * 2, device=x.device, dtype=torch.float64)
        stats = torch.empty(B * G * 2, device=x.device, dtype=torch.float32)
        L.call("sx_groupnorm_fwd", x.data_ptr(), B, Cd, V, G, _ptr(gamma), _ptr(beta), float(eps), csum.data_ptr(),
               stats.data_ptr(), y.data_ptr(), _rt() if round_out else 0, _stream())
        ctx.save_for_backward(x, gamma, stats)
        ctx.meta = (G,)
        ctx.leaves = (gamma, beta)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, stats = ctx.saved_tensors
        (G,) = ctx.meta
        B, Cd, V = x.shape
        dy = dy.contiguous()
        dx = torch.empty_like(x)
        csum = torch.empty(B * Cd * 2, device=x.device, dtype=torch.float64)
        coef = torch.empty(B * G * 2, device=x.device, dtype=torch.float32)
        dg = db = dgb = dbb = None
        if gamma is not None:
            dgb, dg = _sink_or_zeros(ctx.leaves[0])
            dbb, db = _sink_or_zeros(ctx.leaves[1])
        L.call("sx_groupnorm_bwd", dy.data_ptr(), x.data_ptr(), B, Cd, V, G, _ptr(gamma), stats.data_ptr(), csum.data_ptr(),
               coef.data_ptr(), dx.data_ptr(), _ptr(dgb), _ptr(dbb), _stream())
        return dx, dg, db, None, None, None


def conv1x1_add(x, W, b=None, addend=None):
    """x [B,Cin,*sp] -> [B,Cout,*sp]: 1x1(x1) convolution (+ bias) (+ addend of the output's shape)."""
    sp = x.shape[2:]
    B, Cin = x.shape[:2]
    y = _Conv1x1Add.apply(x.reshape(B, Cin, -1), W, b, None if addend is None else addend.reshape(B, W.shape[0], -1))
    return y.view(B, W.shape[0], *sp)


def group_norm(x, gamma, beta, num_groups, eps=1e-5, round_out=False):
    sp = x.shape
    return _GroupNorm.apply(x.reshape(sp[0], sp[1], -1), gamma, beta, int(num_groups), float(eps), round_out).view(sp)


_FPN_FUSION = True


def set_fpn_fusion(on: bool):
    """Switch the fused FPN pyramid stages (conv1x1 + add GEMM, GroupNorm kernels) on or off (off = stock PyTorch modules)."""
    global _FPN_FUSION
    _FPN_FUSION = bool(on)


def fpn_fusion_enabled() -> bool:
    return _FPN_FUSION


def conv1x1_ok(x, conv) -> bool:
    """Whether the tensor-core path can take this 1x1 convolution: TMA needs 16-byte pitches on both operands."""
    V = 1
    for d in x.shape[2:]:
        V *= int(d)
    k = conv.kernel_size
    return x.is_cuda and x.dtype == torch.float32 and all(int(t) == 1 for t in k) and conv.groups == 1 and \
        all(int(t) == 1 for t in conv.stride) and all(int(t) == 0 for t in conv.padding) and \
        V % 4 == 0 and conv.in_channels % 4 == 0


def fpn_stage(cur, higher, conv, norm, scheme="AN"):
    """One bottom-up FPN stage (segtran3d.py:299-313 / :347-359, segtran2d.py:244-257 / :286-300):
        'AN': norm(conv(cur) + upsample(higher))        otherwise: norm(conv(cur)) + upsample(higher)
    conv: nn.Conv2d/3d with a 1x1(x1) kernel, norm: nn.GroupNorm.  The upsampled level is the GEMM epilogue's addend."""
    up_size = tuple(cur.shape[2:])
    hi = higher if tuple(higher.shape[2:]) == up_size else resize_linear(higher, up_size)
    if scheme == 'AN':
        y = conv1x1_add(cur, conv.weight, conv.bias, addend=hi)
        return group_norm(y, norm.weight, norm.bias, norm.num_groups, norm.eps)
    y = conv1x1_add(cur, conv.weight, conv.bias)
    return _Add.apply(group_norm(y, norm.weight, norm.bias, norm.num_groups, norm.eps), hi)


def seg_head(curr, vfeat_fused, grid, Wb, bb, Wc, bc, out_size, d_pool_k=1, permute_dhw_to_hwd=False):
    """Collapsed voxel-wise head.  curr [B,Cf,*sp1]; vfeat_fused [B,N,F] tokens on `grid`;
    3-D: sp1=(D1,H1,W1), depth x d_pool_k, permute to (H,W,D), trilinear to out_size=(H,W,D)  (segtran3d.py:364-496)
    2-D: sp1=(H1,W1), bilinear to out_size=(H,W)                                              (segtran2d.py:304-436)"""
    B, N, Fd = vfeat_fused.shape
    K = Wc.shape[0]
    Wc2 = Wc.reshape(K, Fd)
    sp1 = tuple(curr.shape[2:])
    tv = _TokenClassScores.apply(vfeat_fused, Wc2).view(B, K, *grid)
    tvup = resize_linear(tv, sp1).reshape(B, K, -1)
    Lo = _HeadContract.apply(curr, Wb, bb, Wc2, bc, tvup)
    if len(sp1) == 3:
        if d_pool_k > 1:
            Lo = resize_linear(Lo, (sp1[0] * d_pool_k, sp1[1], sp1[2]))
        H, W, D = out_size
        Lo = resize_linear(Lo, (D, H, W))                  # same maps as interpolating the (H,W,D)-permuted tensor
        Dd = Lo.shape[2]
        out = transpose(Lo.reshape(B * K, Dd, H * W)).view(B, K, H, W, Dd)
        return out
    return resize_linear(Lo, tuple(out_size))


# ------------------------------------------------------------------------------------------------
# attention-consistency loss (train3d.py:426-449, train2d.py:668-723): csrc/sx_consist.cu
# ------------------------------------------------------------------------------------------------
CONSIST_BCE, CONSIST_MARGIN = L.SX_CONSIST_BCE, L.SX_CONSIST_MARGIN


def _consist_pack(x3: torch.Tensor, transpose_in: bool, rnd: int) -> torch.Tensor:
    """[B,R,C] -> K-major [B,N,pad4(A)] copy of the pair operand (N, A) = (R, C), or (C, R) when transpose_in; the pad
    columns are zero (the column sums of the margin variant run over them); TF32-rounded when rnd."""
    B = x3.shape[0]
    N, A = (x3.shape[2], x3.shape[1]) if transpose_in else (x3.shape[1], x3.shape[2])
    Ap = _pad4(A)
    if Ap == A and x3.is_contiguous():
        out = torch.empty((B, N, A), device=x3.device, dtype=torch.float32)
        if transpose_in:
            L.call("sx_transpose", x3.data_ptr(), B, A, N, out.data_ptr(), _stream())
            src = out
        else:
            src = x3
    else:
        out = torch.zeros((B, N, Ap), device=x3.device, dtype=torch.float32)
        out[..., :A].copy_(x3.transpose(1, 2) if transpose_in else x3)
        src = out
    if rnd or src is not out:
        L.call("sx_convert", src.data_ptr(), L.SX_F32, out.numel(), out.data_ptr(), L.SX_F32, rnd, _stream())
    return out


def _consist_colsums(P: torch.Tensor, A: int) -> torch.Tensor:
    """[B,N,Ap] -> [B,A] column sums per batch, in a fixed order."""
    B, N, Ap = P.shape
    cs = _zeros((B, Ap), P.device)
    L.call("sx_colsum_batched", P.data_ptr(), 1, 0, B, N * Ap, N, Ap, Ap, cs.data_ptr(), *_part_args(P.device), _stream())
    return cs if Ap == A else cs[:, :A].contiguous()


class _AttnConsist(torch.autograd.Function):
    """One layer's attention-consistency loss.  Pair entry (Xo [B,1,N,A], Xi [B,1,A,N]): X = Xo Xi is formed tile by tile
    on the tensor cores (precision class "big") and never stored; dense entry X [B,1,N,N].  F [B,K,N] is the flattened
    downsampled mask.  cap: optional device float[2] that accumulates the layers' losses and the 2-D cap factor."""

    @staticmethod
    def forward(ctx, Xo, Xi, X, F, variant, cap, cap_scale):
        _req_cuda(Xo, Xi, X, F, cap)
        B, K, N = F.shape
        dev = F.device
        need = any(ctx.needs_input_grad[:3])
        a = L.sx_consist_args()
        a.B, a.N, a.K, a.variant = B, N, K, variant
        F = F.contiguous()
        a.F = F.data_ptr()
        out = torch.empty(2 + B, device=dev, dtype=torch.float32)
        a.out = out.data_ptr()
        a.cap, a.cap_scale = _ptr(cap), float(cap_scale)
        a.part, a.part_floats = _part_args(dev)
        margin = variant == CONSIST_MARGIN
        nn2 = 1.0 / (float(N) * N)
        saved = []
        if X is None:
            A = Xo.shape[-1]
            three = _three_pass("big")
            XoP = _consist_pack(Xo.reshape(B, N, A), False, 0 if three else 1)
            XtP = _consist_pack(Xi.reshape(B, A, N), True, 0 if three else 1)
            cs_o = cs_t = None
            if margin:                   # mu_b = (1^T Xo_b)(Xi_b 1) / N^2: no pass over X
                cs_o, cs_t = _consist_colsums(XoP, A), _consist_colsums(XtP, A)
                mu = _sgemm(cs_o, cs_t, 1, 1, A, (A, 1), (1, 1), alpha=nn2, Z=B, zs=(A, A, 1)).view(B)
                a.mu = mu.data_ptr()
            ko, kt = (_split_cat(XoP[..., :A], 0)[0], _split_cat(XtP[..., :A], 1)[0]) if three else (XoP, XtP)
            a.A = ko.shape[-1] if three else A
            a.Xo, a.xo_ld, a.xo_bstride = ko.data_ptr(), ko.stride(1), ko.stride(0)
            a.Xt, a.xt_ld, a.xt_bstride = kt.data_ptr(), kt.stride(1), kt.stride(0)
            a.round_r = _rt()
            saved = [XoP, XtP, cs_o, cs_t]
            ctx.shapes = (Xo.shape, Xi.shape, A)
        else:
            X3 = X.reshape(B, N, N)
            if X3.stride(2) != 1 or X3.stride(0) != N * X3.stride(1):
                X3 = X3.contiguous()
            if margin:                   # mu_b: one ordered reduction over the rows of X_b
                rs = _zeros((B * N,), dev)
                L.call("sx_rowsum", X3.data_ptr(), B * N, N, X3.stride(1), B * N, rs.data_ptr(), *_part_args(dev), _stream())
                mu = _zeros((B,), dev)
                L.call("sx_rowsum", rs.data_ptr(), B, N, N, B, mu.data_ptr(), *_part_args(dev), _stream())
                L.call("sx_scale", mu.data_ptr(), B, None, nn2, mu.data_ptr(), _stream())
                a.mu = mu.data_ptr()
            a.X, a.x_ld, a.x_bstride = X3.data_ptr(), X3.stride(1), X3.stride(0)
            ctx.shapes = (X.shape,)
        R = None
        if need:
            R = _rowpad_empty((B, N, N), dev)
            a.R, a.ldr = R.data_ptr(), R.stride(1)
        L.call("sx_attn_consist_fwd", C.byref(a), _stream())
        ctx.save_for_backward(out, R, *[t for t in saved if t is not None])
        ctx.meta = (B, N, variant, X is None, margin)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        out, R, *rest = ctx.saved_tensors
        B, N, variant, pair, margin = ctx.meta
        a = L.sx_consist_args()
        a.B, a.N, a.variant, a.out = B, N, variant, out.data_ptr()
        g = g.contiguous()
        dXo = dXi = dX = None

        def finish(G, rows, cols, vrow, vcol):             # in place: G <- s * (G + m_b v)
            L.call("sx_attn_consist_bwd", C.byref(a), g.data_ptr(), G.data_ptr(), rows, cols, G.stride(-2),
                   G.stride(-3), _ptr(vrow), _ptr(vcol), G.data_ptr(), G.stride(-2), G.stride(-3), _stream())
            return G

        if pair:
            XoP, XtP = rest[0], rest[1]
            cs_o, cs_t = (rest[2], rest[3]) if margin else (None, None)
            xo_shape, xi_shape, A = ctx.shapes
            if ctx.needs_input_grad[0]:              # dXo_b = R_b Xi_b^T
                G = gemm_nt(R, XtP[..., :A].transpose(1, 2), round_out=False)[0]
                dXo = finish(G, N, A, None, cs_t).view(xo_shape)
            if ctx.needs_input_grad[1]:              # dXi_b = Xo_b^T R_b
                G = gemm_nt(XoP[..., :A].transpose(1, 2), R.transpose(1, 2), round_out=False)[0]
                dXi = finish(G, A, N, cs_o, None).view(xi_shape)
        elif ctx.needs_input_grad[2]:
            (x_shape,) = ctx.shapes
            dX = torch.empty((B, N, N), device=R.device, dtype=torch.float32)
            L.call("sx_attn_consist_bwd", C.byref(a), g.data_ptr(), R.data_ptr(), N, N, R.stride(1), R.stride(0), None,
                   None, dX.data_ptr(), N, N * N, _stream())
            dX = dX.view(x_shape)
        return dXo, dXi, dX, None, None, None, None


class _ClampIf(torch.autograd.Function):
    """The scores a layer keeps for the attention-consistency loss (segtran_shared.py:578-598): clamp(S, -clip, clip) when
    the call's maximum (*amax, on the device) exceeds clip, S otherwise; the clamp mask in the backward."""

    @staticmethod
    def forward(ctx, S, amax, clip):
        R, Lr = S.numel() // S.shape[-1], S.shape[-1]
        if not _rows_ok(S):
            S = _rowpad(S)
        out = _rowpad_empty(S.shape, S.device)
        L.call("sx_clamp_if", S.data_ptr(), R, Lr, S.stride(-2), amax.data_ptr(), float(clip), None, 0, out.data_ptr(),
               out.stride(-2), _stream())
        ctx.save_for_backward(S, amax)
        ctx.clip = float(clip)
        return out

    @staticmethod
    def backward(ctx, dY):
        S, amax = ctx.saved_tensors
        R, Lr = S.numel() // S.shape[-1], S.shape[-1]
        dY = dY if dY.is_contiguous() else _rowpad(dY)
        ldy = Lr if dY.is_contiguous() else dY.stride(-2)
        dS = _rowpad_empty(S.shape, S.device)
        L.call("sx_clamp_if", S.data_ptr(), R, Lr, S.stride(-2), amax.data_ptr(), ctx.clip, dY.data_ptr(), ldy,
               dS.data_ptr(), dS.stride(-2), _stream())
        return dS, None, None


def clamp_if(S, amax, clip):
    return _ClampIf.apply(S, amax, clip)


def attn_consist(entry, F, variant, cap=None, cap_scale=1.0):
    """Attention-consistency loss of one layer entry of `layers_attn_scores` as a 0-dim device tensor.
    entry: [in_ator_scores [B,1,A,N], ator_out_scores [B,1,N,A]] (squeezed layer, X = ator_out . in_ator) or the
    dense [B,1,N,N] scores (--nosqueeze); F [B,K,N] fp32 (K <= 16); variant CONSIST_BCE (train3d.py) or CONSIST_MARGIN
    (train2d.py).  cap (device float[2]): cap[0] += the loss, cap[1] <- the factor 1/t if t = cap_scale*cap[0] > 1, else 1
    — train2d.py's cap on the layer mean, read on the device by the caller."""
    if isinstance(entry, (list, tuple)):
        Xi, Xo = entry
        return _AttnConsist.apply(Xo, Xi, None, F, int(variant), cap, cap_scale)
    return _AttnConsist.apply(None, None, entry, F, int(variant), cap, cap_scale)
