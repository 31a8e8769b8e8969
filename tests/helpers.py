"""Shared test helpers (tolerances, fixture loading, oracle drivers)."""
import os

import torch

from oracle import segtran_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), map_location="cpu", weights_only=False)


def rel_err(a, b):
    """max|a-b| / max|b| — the '1e-3 rel' of BASELINE.json's north_star, as used in every parity test."""
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def rms_rel(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30))


def host_keep(seed, idx, p):
    """Keep mask that the counter-based dropout hash (csrc/sx_common.cuh, restated by oracle/head_oracle.py:drop_keep1)
    draws at the flat element indices idx (int64 tensor) -> bool tensor of idx's shape, on idx's device."""
    import numpy as np
    from oracle.head_oracle import drop_keep1
    keep = drop_keep1(int(seed) & ((1 << 64) - 1), idx.detach().cpu().numpy().astype(np.uint64), p)
    return torch.from_numpy(keep).to(idx.device)


def pitched_index(rows, cols, ld, base=0, device="cuda"):
    """flat element indices of a [rows, cols] view whose rows start ld elements apart, the first at element `base`"""
    r = torch.arange(rows, dtype=torch.int64, device=device)[:, None]
    return base + r * ld + torch.arange(cols, dtype=torch.int64, device=device)[None, :]


# ------------------------------------------------------------------------------------------------
# CUDA kernels against float64 PyTorch
# ------------------------------------------------------------------------------------------------
def close(a, b, tol):
    """max|a - b| / max|b| < tol, b the float64 reference (moved to a's device)"""
    b = b.to(a.device)
    if b.numel() == 0:
        return
    err = float((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30))
    assert err < tol, err


def close_on_scale(a, b, scale, tol):
    """max|a - b| < tol * scale (exact agreement when scale is 0): for sums that cancel, compared on a neighbour's scale"""
    err = float((a.double() - b.to(a.device)).abs().max())
    assert err < tol * scale or (scale == 0 and err == 0), (err, scale)


def run_twice(fn, inputs, seed=1, kernels=()):
    """fn(*leaves) -> output, then backward with a fixed upstream gradient; done twice on fresh leaves.  Asserts that
    both runs agree bit for bit and, if `kernels` is given, that forward + backward launch kernels of those names
    (assert_launched).  Returns (output, [grads]) of the first run."""
    def step():
        leaves = [t.detach().clone().requires_grad_() for t in inputs]
        out = fn(*leaves)
        gen = torch.Generator(device=out.device).manual_seed(seed)
        out.backward(torch.randn(out.shape, device=out.device, generator=gen))
        return out.detach(), [t.grad for t in leaves]
    (o1, g1), (o2, g2) = step(), step()
    assert torch.equal(o1, o2)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)
    if kernels:
        assert_launched(step, *kernels)
    return o1, g1


def reference(fn, inputs, out_shape, seed=1):
    """fp64 output and gradients of fn on the same inputs and upstream gradient as run_twice."""
    leaves = [t.detach().double().requires_grad_() for t in inputs]
    out = fn(*leaves)
    gen = torch.Generator(device=out.device).manual_seed(seed)
    out.backward(torch.randn(out_shape, device=out.device, generator=gen).double())
    return out.detach(), [t.grad for t in leaves]


def prologue64(x, g, b, pe, posw, mask=None, keep=None, p=0.0):
    """h = mask * dropout(LN(LN_{g,b}(x) + posw * pe[..., :C])) (pe None: no positional code, no second LayerNorm);
    mask [rows] of 0/1, keep (x's shape) the dropout's keep mask"""
    import torch.nn.functional as F
    C = x.shape[-1]
    t = F.layer_norm(x, (C,), g, b, 1e-12)
    if pe is not None:
        t = F.layer_norm(t + posw * pe[..., :C], (C,), None, None, 1e-12)
    if mask is not None:
        t = t * mask.view(*x.shape[:-1], 1).to(t)
    return t if keep is None else t * keep / (1 - p)


def ln_softaggr64(Y, g, b, ws, bs, keep=None, p=0.0):
    """out = sum_m softmax_m(Yn_m . ws + bs) Yn_m, Yn = LN_{g,b}(dropout(Y)), Y [B, M, N, F]"""
    import torch.nn.functional as F
    if keep is not None:
        Y = Y * keep / (1 - p)
    yn = F.layer_norm(Y, (Y.shape[-1],), g, b, 1e-12)
    return (yn * torch.softmax(F.linear(yn, ws, bs), dim=1)).sum(1)


# ------------------------------------------------------------------------------------------------
# which kernels ran: torch.profiler sessions bracketed by sentinel kernels
# ------------------------------------------------------------------------------------------------
SENTINEL = "spin_kernel"          # the kernel of torch.cuda._sleep; no library op launches it
VOID_SESSIONS = [0]               # sessions discarded because a sentinel's record was lost


def cuda_kernels(fn, reps=2):
    """(names of the CUDA kernels a profiler session recorded while fn() ran `reps` times, spaces removed; whether the
    record is complete).  The session launches a sentinel kernel before and one after fn's launches, each followed by a
    synchronize: a session that lost the record of either sentinel lost records around fn too, and is reported as
    incomplete (on an H100 with torch 2.11, a process that has done much CUDA work sometimes loses records of a session)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
    counts = {e.key.replace(" ", ""): e.count for e in prof.key_averages()}
    sentinels = sum(c for k, c in counts.items() if SENTINEL in k)
    return sorted(counts), sentinels == 2


def assert_launched(fn, *wanted, tries=6):
    """fn() launches, for each string in `wanted`, a kernel whose name contains it: the dispatch branch it names was
    taken.  fn must be repeatable.  A complete session (both sentinels recorded) decides; an incomplete one is void
    and is run again.  When every session is void the branch cannot be observed in this process, and the test is
    reported as skipped (its numeric checks, which run before this one, have passed): a lost record is never taken for
    a wrong branch, nor a wrong branch for a pass."""
    import pytest
    for _ in range(tries):
        names, complete = cuda_kernels(fn)
        if complete:
            missing = [w for w in wanted if not any(w in n for n in names)]
            assert not missing, "no kernel %s among %s" % (missing, names)
            return
        VOID_SESSIONS[0] += 1
    pytest.skip("numeric checks passed; kernel-name check undecided: the profiler lost the sentinel records of %d "
                "sessions in a row (%s)" % (tries, ", ".join(wanted)))


def oracle_encoder(fx, x=None, dtype=torch.float32, collect=None):
    p = {"voxel_fusion." + k: v.to(dtype) for k, v in fx["state_dict"].items()}
    x = fx["x"] if x is None else x
    return O.fusion_encoder(p, "voxel_fusion.", x.to(dtype), fx["voxels_pos"].to(dtype), fx["vmask"], fx["dims"],
                            fx["num_modes"], collect=collect, **variant_kwargs(fx)), p


def variant_kwargs(fx):
    return dict(use_squeezed_transformer=fx.get("use_squeezed_transformer", True),
                has_FFN_in_squeeze=fx.get("has_FFN_in_squeeze", False),
                trans_output_type=fx.get("trans_output_type", "private"))


def encoder_config(cfg_cls, *, dims, num_modes=4, num_attractors=16, pos_dim=3, qk_have_bias=True, dropout=0.0):
    """SegtranConfig (reference's or ours) with what Segtran{2d,3d}Config.update_config would derive."""
    cfg = cfg_cls()
    cfg.num_translayers = len(dims) - 1
    cfg.translayer_dims = list(dims)
    cfg.translayer_compress_ratios = [1] * len(dims)
    cfg.trans_in_dim, cfg.trans_out_dim, cfg.min_feat_dim = dims[0], dims[-1], min(dims)
    cfg.num_modes, cfg.num_attractors, cfg.pos_dim, cfg.qk_have_bias = num_modes, num_attractors, pos_dim, qk_have_bias
    cfg.hidden_dropout_prob = cfg.attention_probs_dropout_prob = dropout
    return cfg


def build_b200_encoder(fx, device="cuda", dropout=0.0):
    import segtran_b200.networks.segtran_shared as S
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"],
                         num_attractors=fx["num_attractors"], pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"],
                         dropout=dropout)
    cfg.use_squeezed_transformer = fx.get("use_squeezed_transformer", True)
    cfg.has_FFN_in_squeeze = fx.get("has_FFN_in_squeeze", False)
    cfg.trans_output_type = fx.get("trans_output_type", "private")
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.tie_qk)
    enc.load_state_dict(fx["state_dict"], strict=True)
    return enc.to(device)


class AffinePickNet(torch.nn.Module):
    """Stand-in segmentation net for the inference-path fixtures: class k's score = a[k] * x[:, ch[k]] + b[k] — element-wise, so
    it is reproducible to the last ulp on any device (the sliding-window logic is what the fixtures pin, not a network)."""

    def __init__(self, a, b, ch):
        super().__init__()
        self.a, self.b, self.ch = [float(v) for v in a], [float(v) for v in b], [int(c) for c in ch]

    def forward(self, x):
        return torch.stack([x[:, c] * a + b for a, b, c in zip(self.a, self.b, self.ch)], dim=1)
