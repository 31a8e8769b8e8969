"""Time one plain-attention (--nosqueeze) encoder layer, forward + backward, with sliding-window positional biases
(--pos bias) and with the learnable sinusoid code (--pos lsinu), alternating the two in one process.

    python tools/time_posbias.py [--iters 30] [--warmup 5] [--rounds 5]

Shapes: 2-D cfg 1 (36x36 tokens, C = 1792, 4 modes, batch 2) and 3-D (14x14x14 tokens, C = 1024, 4 modes, batch 4).
Prints the device name and its power limit next to the numbers (they are part of the measurement)."""
import argparse
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import segtran_b200.networks.segtran_shared as S  # noqa: E402


def build(pos, grid, C):
    cfg = S.SegtranConfig()
    cfg.num_translayers = 1
    cfg.translayer_dims = [C, C]
    cfg.translayer_compress_ratios = [1, 1]
    cfg.trans_in_dim = cfg.trans_out_dim = cfg.min_feat_dim = C
    cfg.num_modes, cfg.pos_dim = 4, len(grid)
    cfg.use_squeezed_transformer = False
    cfg.pos_code_type = pos
    cfg.max_pos_size = grid
    torch.manual_seed(0)
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.init_weights)
    enc.apply(init.tie_qk)
    enc.apply(init.add_identity_bias)
    return enc.cuda().train()


def time_one(enc, grid, B, C, iters, warmup):
    N = math.prod(grid)
    x = torch.randn(B, N, C, device="cuda", requires_grad=True)
    pos = torch.stack(torch.meshgrid(*[torch.arange(g) for g in grid], indexing="ij"), -1).reshape(1, N, len(grid))
    pos = pos.float().cuda().expand(B, N, len(grid))
    vm = torch.ones(B, N, 1, device="cuda")
    shape = torch.Size(grid)

    def step():
        y = enc(x, pos, vm, shape)
        y.sum().backward()

    for _ in range(warmup):
        step()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                    # noqa: BLE001  (no nvidia-smi: report it as unknown)
        pl = "unknown"
    print("device: %s, power limit: %s" % (name, pl))
    for label, grid, C, B in (("2-D 36x36 C=1792 B=2", (36, 36), 1792, 2), ("3-D 14^3 C=1024 B=4", (14, 14, 14), 1024, 4)):
        encs = {p: build(p, grid, C) for p in ("lsinu", "bias")}
        res = {p: [] for p in encs}
        for _ in range(args.rounds):
            for p, enc in encs.items():
                res[p].append(time_one(enc, grid, B, C, args.iters, args.warmup))
        print("%s  fwd+bwd ms per layer:  lsinu %s   bias %s" % (
            label, " / ".join("%.3f" % t for t in res["lsinu"]), " / ".join("%.3f" % t for t in res["bias"])))
        del encs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
