"""Time one --nosqueeze layer, forward + backward, in three variants alternated in one process, and check that they agree:
  multihead  --multihead on this build (MultiHeadFeatTrans on the fused attention kernel);
  multimode  the default multi-mode expansion on this build (ExpandedFeatTrans, fused squeeze-out node);
  eager      the multi-head layer in the reference's formulation (oracle/multihead_oracle.py) in eager fp32 PyTorch on the
             same GPU (TF32 matmuls off), with the multihead layer's weights.

    python tools/time_multihead.py [--iters 10] [--warmup 3] [--rounds 5]

Shapes: cfg 1 (2-D 36x36 tokens, C = F = 1792, 4 heads of dh = 448, batch 2) and cfg 4 (3-D 14x14x14 tokens, C = F = 1024,
4 heads of dh = 256, batch 4).  Prints the device name and its power limit next to the numbers (they are part of the
measurement), the per-round times and their median, and the multihead output's max|a-b|/max|b| against eager."""
import argparse
import math
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import segtran_b200.networks.segtran_shared as S  # noqa: E402
from oracle import multihead_oracle as MH  # noqa: E402


def build(multihead, grid, C):
    cfg = S.SegtranConfig()
    cfg.num_translayers = 1
    cfg.translayer_dims = [C, C]
    cfg.translayer_compress_ratios = [1, 1]
    cfg.trans_in_dim = cfg.trans_out_dim = cfg.min_feat_dim = C
    cfg.num_modes, cfg.pos_dim = 4, len(grid)
    cfg.use_squeezed_transformer = False
    cfg.ablate_multihead = multihead
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_multihead.py measures on the GPU; no CUDA device is available")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                    # noqa: BLE001  (no nvidia-smi: report it as unknown)
        pl = "unknown"
    print("device: %s, power limit: %s" % (name, pl))
    for label, grid, C, B in (("cfg 1: 2-D 36x36 C=F=1792 B=2", (36, 36), 1792, 2),
                              ("cfg 4: 3-D 14^3 C=F=1024 B=4", (14, 14, 14), 1024, 4)):
        N = math.prod(grid)
        torch.manual_seed(1)
        x = torch.randn(B, N, C, device="cuda", requires_grad=True)
        pos = torch.stack(torch.meshgrid(*[torch.arange(g) for g in grid], indexing="ij"), -1).reshape(1, N, len(grid))
        pos = pos.float().cuda().expand(B, N, len(grid)).contiguous()
        vm = torch.ones(B, N, 1, device="cuda")
        shape = torch.Size(grid)
        mh, mm = build(True, grid, C), build(False, grid, C)
        p = {k: v.detach().clone().requires_grad_() for k, v in mh.state_dict().items() if ".key." not in k}

        def run_mh():
            y = mh(x, pos, vm, shape)
            y.sum().backward()
            return y

        def run_mm():
            y = mm(x, pos, vm, shape)
            y.sum().backward()
            return y

        def run_eager():
            y = MH.fusion_encoder_multihead(p, "", x, pos, vm, [C, C], 4)
            y.sum().backward()
            return y

        # agreement of the outputs: eval mode (the timed steps run with the config's default dropout of 0.1)
        mh.eval()
        with torch.no_grad():
            e = float((mh(x, pos, vm, shape) - MH.fusion_encoder_multihead(p, "", x, pos, vm, [C, C], 4)).abs().max())
            ref_max = float(MH.fusion_encoder_multihead(p, "", x, pos, vm, [C, C], 4).abs().max())
        mh.train()
        variants = {"multihead": run_mh, "multimode": run_mm, "eager": run_eager}
        res = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                res[k].append(_events(fn, args.iters, args.warmup))
        print("%s  (multihead vs eager output, eval mode: max-rel %.2e)" % (label, e / ref_max))
        for k, ts in res.items():
            print("    %-10s fwd+bwd ms per layer: median %.3f   rounds %s" % (
                k, statistics.median(ts), " / ".join("%.3f" % t for t in ts)))
        del mh, mm, p, x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
