"""Time the 3-D training loop's batch preparation (train3d.py:711-715: brats_map_label, then RandomResizedCrop with
--randscale 0.1) as the library's kernels against the eager PyTorch formulation on the same GPU.

    python tools/time_prep3d.py [--rounds 9] [--iters 20] [--steps 10] [--json out.json]

Workload: the BraTS batch of the published result, volume [4,4,112,112,96] fp32 and uint8 labels [4,112,112,96]
(n-hot mask [4,4,112,112,96] fp32, 19.3 MB like the volume), with two fixed crop records, one per branch of the crop:
scale 0.9 (intermediate [101,101,86], zero-padded) and scale 1.1 (intermediate [123,123,105], cropped).
  * eager: oracle/prep3d_oracle.py in float32, the reference's formulation (four boolean-mask fills into a zeroed
    [K,B,...] buffer and a permuted view; F.interpolate of both tensors, F.pad, two slice clones) with the draws given;
  * segtran_b200: datasets3d.brats_map_label and RandomResizedCrop with the same record on the device.
Each arm is timed per call with CUDA events over --rounds rounds of --iters calls after warm-up: median and spread
(min, max), the peak memory above the inputs (max_memory_allocated), and bytes/s against a byte model from the shapes
(inputs read once, outputs written once).  The two arms' outputs are compared.
Then a captured cfg-4 training step (bench.py's Segtran3d 112^3 x 4 ch, bs 4, 1024 attractors, with fixed features
standing in for the backbone and FlatBertAdam) whose loss reads the prepared n-hot mask, timed two ways over --steps
replays per round: the preparation (drop-ins, device draws) run eagerly before each replay, and inside the graph.
The device name and power limit are read in the same run.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPE = (112, 112, 96)
B, CV, K = 4, 4, 4


def timed(fn, rounds, iters, warmup=3):
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


def arm(fn, rounds, iters, nbytes):
    """Per-call time, bytes/s of the byte model, and the peak memory allocated above what was live before."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    t = timed(fn, rounds, iters)
    t["GB_per_s"] = nbytes / (t["median_ms"] * 1e-3) / 1e9
    t["peak_extra_MB"] = peak / 1e6
    return t


def record(scale):
    s = float(torch.tensor(scale, dtype=torch.float32))
    padded = [max(int(torch.tensor(float(L)) * s), L) for L in SHAPE]
    return torch.tensor([s, s, s] + [(p - L) // 2 for p, L in zip(padded, SHAPE)], dtype=torch.float32)


def captured_step(a, rep):
    """bench.py's cfg-4 step with the batch preparation before it, eager or captured with it."""
    import bench
    from segtran_b200 import ops
    from segtran_b200.datasets3d import RandomResizedCrop, brats_map_label
    from segtran_b200.graph import CapturedStep
    from segtran_b200.parallel import GradBucket
    from segtran_b200.train import FlatBertAdam, seg_loss
    c = bench.CONFIGS[4]
    dev = torch.device("cuda", torch.cuda.current_device())
    net = bench.build_net(c, "cuda").to(dev).train()
    hp = bench.hot_params(net, c)
    bucket = GradBucket(hp, direct_accumulate=True)
    feat, curr, _ = bench.synthetic_batch(c, c["B"], dev, 4242)
    feat.requires_grad_()
    curr.requires_grad_()
    pw, cw = bench.loss_weights(c, dev)
    T = bench.TRAIN
    opt = FlatBertAdam([{"params": hp, "lr": T["lr"], "weight_decay": T["decay"]}], warmup=T["warmup"],
                       t_total=T["t_total"], grad_clip=T["grad_clip"], bucket=bucket)
    sp = (c["S"],) * 3
    g = torch.Generator().manual_seed(7)
    volume = torch.randn((c["B"], 4) + sp, generator=g).to(dev)
    labels = torch.randint(0, 4, (c["B"],) + sp, generator=g, dtype=torch.uint8).to(dev)
    cp = (-0.1, 0.1)
    prepared = {}

    def prepare():
        mask = brats_map_label(labels, False)
        prepared["v"], prepared["m"] = RandomResizedCrop(volume, mask, sp, cp)

    def compute(with_prep):
        def fn():
            if with_prep:
                prepare()
            bucket.zero()
            feat.grad = None
            curr.grad = None
            logits = net.hot_path(feat, curr, None, sp)
            loss, _, _ = seg_loss(logits, prepared["m"], pw, cw, T["dice_w"])
            loss.backward()
            opt.step()
            return loss
        return fn

    prepare()                                                   # static mask buffer for the eager-preparation graph
    static_m = prepared["m"]
    g_outside = CapturedStep(compute(False), warmup=2)

    def outside():
        ops.advance_seed(dev)
        prepare()
        static_m.copy_(prepared["m"])                           # the graph reads its captured mask buffer
        prepared["m"] = static_m
        g_outside()

    g_inside = CapturedStep(compute(True), warmup=2)

    def inside():
        ops.advance_seed(dev)
        g_inside()

    rep["captured_cfg4_step"] = dict(
        workload="bench.py cfg 4 step (hot path + seg_loss + backward + FlatBertAdam), batch [4,4,112,112,112], the loss "
                 "on the prepared mask; the volume crop is computed, the fixed features stand in for the backbone",
        prep_eager_then_replay=timed(outside, a.rounds, a.steps), prep_inside_graph=timed(inside, a.rounds, a.steps),
        launches_in_graph=g_inside.kernel_launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_prep3d: needs a CUDA device")
    from oracle import prep3d_oracle as PO
    from segtran_b200.datasets3d import RandomResizedCrop, brats_map_label

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    rep = dict(device=q, workload="volume [4,4,112,112,96] fp32, uint8 labels [4,112,112,96], --randscale 0.1")
    g = torch.Generator().manual_seed(0)
    volume = torch.randn((B, CV) + SHAPE, generator=g).cuda()
    labels = torch.randint(0, 5, (B,) + SHAPE, generator=g, dtype=torch.uint8).cuda()
    V = SHAPE[0] * SHAPE[1] * SHAPE[2]
    map_bytes = B * V * (1 + 4 * K)
    crop_bytes = 2 * B * (CV + K) * V * 4
    mask_ref = PO.brats_map_label(labels, False)               # the reference's permuted view
    mask = brats_map_label(labels, False)
    rep["brats_map_label"] = dict(
        byte_model_MB=map_bytes / 1e6,
        eager=arm(lambda: PO.brats_map_label(labels, False), a.rounds, a.iters, map_bytes),
        segtran_b200=arm(lambda: brats_map_label(labels, False), a.rounds, a.iters, map_bytes),
        equal=bool(torch.equal(mask, mask_ref)))
    for scale in (0.9, 1.1):
        rec = record(scale)
        rec_dev = rec.cuda()
        ev, em = PO.resized_crop(volume, mask_ref, SHAPE, rec)
        ov, om = RandomResizedCrop(volume, mask_ref, SHAPE, (-0.1, 0.1), draws=rec_dev)
        rep["RandomResizedCrop_scale_%.1f" % scale] = dict(
            record=rec.tolist(), byte_model_MB=crop_bytes / 1e6,
            eager=arm(lambda: PO.resized_crop(volume, mask_ref, SHAPE, rec), a.rounds, a.iters, crop_bytes),
            segtran_b200=arm(lambda: RandomResizedCrop(volume, mask_ref, SHAPE, (-0.1, 0.1), draws=rec_dev),
                             a.rounds, a.iters, crop_bytes),
            max_abs_diff=max(float((ov - ev).abs().max()), float((om - em).abs().max())))
        rep["block_scale_%.1f" % scale] = dict(
            byte_model_MB=(map_bytes + crop_bytes) / 1e6,
            eager=arm(lambda: PO.resized_crop(volume, PO.brats_map_label(labels, False), SHAPE, rec), a.rounds,
                      a.iters, map_bytes + crop_bytes),
            segtran_b200=arm(lambda: RandomResizedCrop(volume, brats_map_label(labels, False), SHAPE, (-0.1, 0.1),
                                                       draws=rec_dev), a.rounds, a.iters, map_bytes + crop_bytes))
    rep["block_device_draws"] = dict(segtran_b200=arm(
        lambda: RandomResizedCrop(volume, brats_map_label(labels, False), SHAPE, (-0.1, 0.1)), a.rounds, a.iters,
        map_bytes + crop_bytes))
    del volume, labels, mask, mask_ref
    torch.cuda.empty_cache()
    captured_step(a, rep)
    out = json.dumps(rep, indent=1)
    print(out)
    if a.json:
        with open(a.json, "w") as f:
            f.write(out)


if __name__ == "__main__":
    main()
