"""Time one mince-transformer layer (--mince --nosqueeze --pos bias), forward + backward, alternating in one process with
the plain --nosqueeze --pos bias layer, and the token-grid resampling kernels on their own.

    python tools/time_mince.py [--iters 30] [--warmup 5] [--rounds 5]

Shapes: 3-D 14x14x14 tokens, C = 1024, 4 modes, batch 4, scales [1,2,4]; 2-D 36x36 tokens, C = 1792, 4 modes, batch 2,
scales [1,2,3]; channel proportions equal.  The resampling rate is the least traffic of a call (the channel windows read
once plus the output written once, bytes from the shapes) over its time, against the H100 SXM data-sheet 3.35 TB/s.
Prints the device name and its power limit next to the numbers (they are part of the measurement)."""
import argparse
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import segtran_b200.networks.segtran_shared as S  # noqa: E402
from segtran_b200 import ops  # noqa: E402

HBM_GBS = 3350.0


def build(mince, grid, C, scales):
    cfg = S.SegtranConfig()
    cfg.num_translayers = 1
    cfg.translayer_dims = [C, C]
    cfg.translayer_compress_ratios = [1, 1]
    cfg.trans_in_dim = cfg.trans_out_dim = cfg.min_feat_dim = C
    cfg.num_modes, cfg.pos_dim = 4, len(grid)
    cfg.use_squeezed_transformer = False
    cfg.pos_code_type = "bias"
    cfg.max_pos_size = grid
    cfg.use_mince_transformer = mince
    cfg.mince_scales = list(scales) if mince else None
    cfg.mince_channel_props = [1] * len(scales) if mince else None
    torch.manual_seed(0)
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.init_weights)
    enc.apply(init.tie_qk)
    enc.apply(init.add_identity_bias)
    return enc.cuda().train()


def _events(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def time_layer(enc, grid, B, C, iters, warmup):
    N = math.prod(grid)
    x = torch.randn(B, N, C, device="cuda", requires_grad=True)
    pos = torch.stack(torch.meshgrid(*[torch.arange(g) for g in grid], indexing="ij"), -1).reshape(1, N, len(grid))
    pos = pos.float().cuda().expand(B, N, len(grid))
    vm = torch.ones(B, N, 1, device="cuda")
    shape = torch.Size(grid)

    def step():
        y = enc(x, pos, vm, shape)
        y.sum().backward()

    return _events(step, iters, warmup)


def time_resampling(grid, B, C, scales, iters, warmup):
    """-> {name: (ms, GB/s)} for the Q (or K) downsampling of all scales and the upsampling of all scales into U."""
    M = 4
    d = C // M
    N = math.prod(grid)
    grids = S.mince_grids(grid, scales)
    idx, _ = S.fracs_to_indices(d, [1] * len(scales))
    wins = [(idx[s], idx[s + 1]) for s in range(len(scales))]
    ratios = [(ops.down_ratio(sc),) * len(grid) for sc in scales]
    q = torch.randn(B, N, C, device="cuda")
    pads = [ops._pad4(b - a) for a, b in wins]
    res = {}
    with torch.no_grad():
        t = _events(lambda: ops.resize_tokens(q, M, grid, grids, ratios, wins), iters, warmup)
        byt = 4 * B * M * (N * d + sum(math.prod(g) * p for g, p in zip(grids, pads)))
        res["downsample Q (all scales)"] = (t, byt / t / 1e6)
        fidx, _ = S.fracs_to_indices(C, [1] * len(scales))           # F = C here
        fwins = [(fidx[s], fidx[s + 1]) for s in range(len(scales))]
        us = [torch.randn(B, M, math.prod(g), ops._pad4(b - a), device="cuda") for g, (a, b) in zip(grids, fwins)]
        t = _events(lambda: ops.resize_tokens_into(us, grid, grids, fwins, C), iters, warmup)
        byt = 4 * (sum(u.numel() for u in us) + B * M * N * C)
        res["upsample P.V into U (all scales)"] = (t, byt / t / 1e6)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_mince.py measures on the GPU; no CUDA device is available")
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                    # noqa: BLE001  (no nvidia-smi: report it as unknown)
        pl = "unknown"
    print("device: %s, power limit: %s" % (name, pl))
    for label, grid, C, B, scales in (("3-D 14^3 C=1024 B=4 scales [1,2,4]", (14, 14, 14), 1024, 4, [1, 2, 4]),
                                      ("2-D 36x36 C=1792 B=2 scales [1,2,3]", (36, 36), 1792, 2, [1, 2, 3])):
        encs = {"plain": build(False, grid, C, scales), "mince": build(True, grid, C, scales)}
        res = {k: [] for k in encs}
        for _ in range(args.rounds):
            for k, enc in encs.items():
                res[k].append(time_layer(enc, grid, B, C, args.iters, args.warmup))
        print("%s  fwd+bwd ms per layer:  plain %s   mince %s" % (
            label, " / ".join("%.3f" % t for t in res["plain"]), " / ".join("%.3f" % t for t in res["mince"])))
        del encs
        torch.cuda.empty_cache()
        for k, (t, gbs) in time_resampling(grid, B, C, scales, args.iters * 4, args.warmup).items():
            print("    %-34s %.4f ms  %7.1f GB/s  (%.1f %% of %.0f GB/s)" % (k, t, gbs, 100 * gbs / HBM_GBS, HBM_GBS))


if __name__ == "__main__":
    main()
