"""Time the 2.5-D model's CUDA segment against the reference formulation on the same GPU.

    python tools/time_segtran25d.py [--batch 2] [--rounds 7] [--iters 5] [--json out.json]

Workload: input [B,4,112,112,96], eff-b3 feature widths, --infpn 34 --outfpn 1234, stemconv, --upd conv, 1024
attractors (9408 tokens x 1536 channels), with a stand-in backbone returning seeded per-slice features, so both arms
start from the same backbone output:
  * segtran_b200: Segtran25d.forward after the backbone: slice-major in-FPN, depth pooling, the encoder, the slice-major
    out-FPN (ops.fpn_stage(slices=96), sx_groupnorm_slices_*) and the collapsed head;
  * eager: oracle/seg25d_oracle.py, the reference's formulation (permuted volumes, the full [B,1536,56,56,96] out-FPN map),
    stock PyTorch fp32 with PyTorch's default TF32 settings.
Forward and forward + backward are timed with CUDA events over --rounds rounds of --iters calls after warm-up; the report
gives the median and the spread (min, max) of the per-call time, the peak memory of each arm (max_memory_allocated, "OOM"
if an arm does not fit), the agreement of the two arms' logits, and the per-launch time and algorithmic bytes/s
(read x twice, write y once) of the slice GroupNorm against nn.GroupNorm on the permuted [B,C,56,56,96] tensor.  The
device name and power limit are read in the same run.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from argparse import Namespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class FixedFeat(torch.nn.Module):
    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def extract_endpoints(self, x):
        return {'reduction_%d' % (i + 1): f for i, f in enumerate(self.feats)}


def build(B, seed=0):
    import segtran_b200.networks.segtran25d as M
    args = Namespace(in_fpn_layers='34', out_fpn_layers='1234', in_fpn_scheme='AN', out_fpn_scheme='AN',
                     translayer_compress_ratios=[1, 1], orig_in_channels=4, inchan_to3_scheme='stemconv',
                     use_pretrained=False, device='cuda', dropout_prob=0.0)
    cfg = M.Segtran25dConfig()
    cfg.update_config(args)
    g = torch.Generator().manual_seed(seed)
    H, W, D = 112, 112, 96
    dims = cfg.bb_feat_dims
    feats = [torch.zeros(1, device="cuda").expand(B * D, dims[0], H, W)] + \
        [torch.randn(B * D, dims[i], H >> i, W >> i, generator=g).cuda().requires_grad_() for i in range(1, 5)]
    torch.manual_seed(seed)
    net = M.Segtran25d(cfg, backbone=FixedFeat(feats)).cuda().eval()
    batch = torch.randn(B, 4, H, W, D, generator=g)
    batch[..., :8] = 0
    return cfg, net, feats, batch.cuda()


def timed(fn, rounds, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    per_call = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        per_call.append(a.elapsed_time(b) / iters)
    return dict(median_ms=statistics.median(per_call), min_ms=min(per_call), max_ms=max(per_call))


def arm(fn, rounds, iters):
    """Time fn and record its peak memory; 'OOM' if it does not fit."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    try:
        t = timed(fn, rounds, iters)
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        return "OOM"
    t["peak_mem_GB"] = torch.cuda.max_memory_allocated() / 1e9
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_segtran25d: needs a CUDA device")
    from oracle import seg25d_oracle as SO
    from segtran_b200 import ops

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    B = a.batch
    cfg, net, feats, batch = build(B)
    G = torch.randn(B, cfg.num_classes, 112, 112, 96, device="cuda")
    p = net.state_dict(keep_vars=True)
    mask = SO.get_mask(batch, 8)
    okw = dict(in_layers=net.in_fpn_layers, out_layers=net.out_fpn_layers, translayer_dims=net.translayer_dims,
               num_modes=cfg.num_modes, D_pool_K=2, upd='conv')

    def ours_fwd():
        with torch.no_grad():
            return net(batch)

    def ours_fb():
        (net(batch) * G).sum().backward()

    def eager_fwd():
        with torch.no_grad():
            return SO.forward(p, feats, mask, B, (112, 112, 96), **okw)

    def eager_fb():
        (SO.forward(p, feats, mask, B, (112, 112, 96), **okw) * G).sum().backward()

    rep = dict(device=q, batch=B, workload="Segtran25d [B,4,112,112,96] eff-b3 infpn 34 / outfpn 1234 stemconv "
                                          "--upd conv, 1024 attractors, 9408 tokens x 1536 ch, backbone excluded")
    rep["segtran_b200"] = dict(fwd=arm(ours_fwd, a.rounds, a.iters), fwd_bwd=arm(ours_fb, a.rounds, a.iters))
    rep["eager"] = dict(fwd=arm(eager_fwd, a.rounds, a.iters), fwd_bwd=arm(eager_fb, a.rounds, a.iters))
    try:
        y, ref = ours_fwd(), eager_fwd()
        rep["logits_max_rel_diff"] = float((y - ref).abs().max() / ref.abs().max())
    except torch.cuda.OutOfMemoryError:
        rep["logits_max_rel_diff"] = "OOM"
    del feats, net, p
    torch.cuda.empty_cache()

    # the out-FPN's GroupNorm at this shape: level 2 (48 channels) at 56x56 on 96 slices per sample
    C, Hs, D = 48, 56, 96
    x = torch.randn(B * D, C, Hs, Hs, device="cuda")
    gn = torch.nn.GroupNorm(8, C).cuda()
    xv = x.view(B, D, C, Hs, Hs).permute(0, 2, 3, 4, 1)               # the reference's [B,C,H,W,D] view
    xc = xv.contiguous()
    nbytes = 3 * x.numel() * 4
    gnrep = {}
    with torch.no_grad():
        for name, fn in (("sx_groupnorm_slices", lambda: ops.group_norm(x, gn.weight, gn.bias, 8, gn.eps, slices=D)),
                         ("nn.GroupNorm_permuted_view", lambda: gn(xv)),
                         ("nn.GroupNorm_contiguous_volume", lambda: gn(xc))):
            t = timed(fn, a.rounds, 20)
            t["GB_per_s"] = nbytes / (t["median_ms"] * 1e-3) / 1e9
            gnrep[name] = t
    rep["groupnorm_fwd_per_launch"] = gnrep
    out = json.dumps(rep, indent=1)
    print(out)
    if a.json:
        with open(a.json, "w") as f:
            f.write(out)


if __name__ == "__main__":
    main()
