"""Time the attention-consistency loss at cfg-4 shapes (B = 4, N = 14^3 = 2744, A = 1024, K = 4): forward plus backward
of the fused kernel path (segtran_b200.train.attn_consist_loss3d / 2d) against the reference formulation run as eager
fp32 PyTorch with TF32 off (X = Xo @ Xi and the [B,N,N] target matrix materialised), alternating the two in one process
over several rounds.  Reports the time per call, the achieved TFLOP/s from shapes (2*B*N^2*A per product: one forward,
two backward) and the peak memory of each; then the fused path's time per C-ABI entry point (CUDA events around each
call, in a run of its own), and the time of an encoder step with --attnconsist on the modules (SegtranFusionEncoder at
cfg-4 shapes, one squeezed layer of width 1024: forward, loss, backward) with either loss.

    python tools/time_attn_consist.py [--rounds 5] [--iters 10]

Prints the device name and its power limit next to the numbers (they are part of the measurement)."""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from segtran_b200 import _lib, train  # noqa: E402
import segtran_b200.networks.segtran_shared as S  # noqa: E402


def eager3d(layers, shape, mask):
    mask = mask.permute(0, 1, 4, 2, 3)
    fm = F.interpolate(mask, size=shape, mode='trilinear', align_corners=False)
    fm = fm.view(fm.size(0), fm.size(1), -1)
    c = torch.clip(torch.matmul(fm.transpose(-2, -1), fm), 0, 1)
    xi, xo = layers[0]
    return F.binary_cross_entropy_with_logits(torch.matmul(xo, xi).squeeze(1), c)


def eager2d(layers, shape, mask):
    fm = F.interpolate(mask, size=shape, mode='bilinear', align_corners=False)
    fm = fm.view(fm.size(0), fm.size(1), -1)
    c = torch.clip(torch.matmul(fm.transpose(-2, -1), fm), 0, 1).bool()
    xi, xo = layers[0]
    x = torch.matmul(xo, xi).squeeze(1)
    mu = x.mean(dim=2, keepdim=True).mean(dim=1, keepdim=True)
    inc = ((x < mu) & c) | ((x > mu - 0.1) & ~c)
    loss = (x - mu)[inc].abs().mean()
    if loss > 1:
        loss = loss / loss.item()
    return loss


def time_one(fn, layers, shape, mask, iters):
    params = [t for e in layers for t in e]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        loss = fn(layers, shape, mask)
        torch.autograd.grad(loss, params)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_attn_consist: needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, check=True).stdout.strip()
    except Exception:                                    # noqa: BLE001  (no nvidia-smi: report it as unknown)
        pl = "unknown"
    print("device: %s, power limit: %s" % (name, pl))
    B, N, A, K, g = 4, 2744, 1024, 4, 14
    flop = 3 * 2.0 * B * N * N * A
    torch.manual_seed(0)
    layers = [[(torch.randn(B, 1, A, N, device="cuda") * 0.05).requires_grad_(),
               (torch.randn(B, 1, N, A, device="cuda") * 0.05).requires_grad_()]]
    lab3 = torch.randint(0, K, (B, 2 * g, 2 * g, 2 * g), device="cuda")
    mask3 = F.one_hot(lab3, K).permute(0, 4, 1, 2, 3).float().contiguous()
    # 2-D at the same N and A: a 49 x 56 token grid
    lab2 = torch.randint(0, K, (B, 98, 112), device="cuda")
    mask2 = F.one_hot(lab2, K).permute(0, 3, 1, 2).float().contiguous()
    cases = [("3d", train.attn_consist_loss3d, eager3d, (g, g, g), mask3),
             ("2d", train.attn_consist_loss2d, eager2d, (49, 56), mask2)]
    for tag, fused, eager, shape, mask in cases:
        for fn in (fused, eager):                          # warm-up of every shape
            time_one(fn, layers, shape, mask, 2)
        res = {"fused": [], "eager": []}
        for _ in range(args.rounds):
            res["fused"].append(time_one(fused, layers, shape, mask, args.iters))
            res["eager"].append(time_one(eager, layers, shape, mask, args.iters))
        for k, v in res.items():
            ms = sorted(t for t, _ in v)
            med = ms[len(ms) // 2]
            print("%s %-5s fwd+bwd: median %.3f ms (rounds %s), %.1f TFLOP/s, peak +%.0f MiB"
                  % (tag, k, med, " ".join("%.3f" % t for t, _ in v), flop / med / 1e9, max(m for _, m in v)))
        print("%s fused, per entry point (ms per call of the loss):" % tag)
        for name, ms in per_call_split(fused, layers, shape, mask, args.iters):
            print("    %-22s %.3f" % (name, ms))
    for r in range(args.rounds):
        t_f = encoder_step(train.attn_consist_loss3d, args.iters)
        t_e = encoder_step(eager3d, args.iters)
        print("encoder step (cfg-4 shapes, --attnconsist, 3-D loss) round %d: fused loss %.3f ms, eager loss %.3f ms"
              % (r, t_f, t_e))


def per_call_split(fn, layers, shape, mask, iters):
    """ms per call of each C-ABI entry point inside one fused forward + backward (events recorded around every call)."""
    rec = []

    class _Ev:
        def __init__(self, name):
            self.name = name

        def __enter__(self):
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

        def __exit__(self, *a):
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            rec.append((self.name, self.e0, e1))

    params = [t for e in layers for t in e]
    _lib.set_hook(lambda name, args: _Ev(name))
    try:
        for _ in range(iters):
            torch.autograd.grad(fn(layers, shape, mask), params)
        torch.cuda.synchronize()
    finally:
        _lib.set_hook(None)
    tot = {}
    for name, e0, e1 in rec:
        tot[name] = tot.get(name, 0.0) + e0.elapsed_time(e1) / iters
    return sorted(tot.items(), key=lambda kv: -kv[1])


def encoder_step(loss_fn, iters, B=4, g=14, C=1024, A=1024, M=4, K=4):
    cfg = S.SegtranConfig()
    cfg.num_translayers, cfg.translayer_dims, cfg.translayer_compress_ratios = 1, [C, C], [1, 1]
    cfg.trans_in_dim = cfg.trans_out_dim = cfg.min_feat_dim = C
    cfg.num_modes, cfg.num_attractors, cfg.pos_dim, cfg.qk_have_bias = M, A, 3, True
    cfg.hidden_dropout_prob = cfg.attention_probs_dropout_prob = 0.0
    cfg.use_attn_consist_loss = True
    torch.manual_seed(0)
    enc = S.SegtranFusionEncoder(cfg, "Fusion").cuda().train()
    N = g ** 3
    x = torch.randn(B, N, C, device="cuda")
    idx = torch.stack(torch.meshgrid(*[torch.arange(g)] * 3, indexing="ij"), -1).view(1, -1, 3).float().cuda() * 8
    vpos = idx.expand(B, -1, -1)
    lab = torch.randint(0, K, (B, 2 * g, 2 * g, 2 * g), device="cuda")
    mask = F.one_hot(lab, K).permute(0, 4, 1, 2, 3).float().contiguous()
    params = [p for p in enc.parameters() if p.requires_grad]

    def step():
        y = enc(x, vpos, None, torch.Size((g, g, g)))
        loss = loss_fn(enc.layers_attn_scores, (g, g, g), mask) + y.mean()
        torch.autograd.grad(loss, params, allow_unused=True)

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


if __name__ == "__main__":
    main()
