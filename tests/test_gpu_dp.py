"""Data-parallel correctness on real GPUs over NCCL (SURVEY §4 item v, reference train3d.py:671-676): a 2-rank step on a
split batch must give the single-GPU gradient of the concatenated batch, and after the BertAdam update every rank must
hold bit-identical parameters.  Needs >= 2 GPUs (skipped otherwise)."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu

TINY = dict(kind="3d", title="tiny 3-D shell", backbone="i3d", B=2, S=16, grid=(4, 4, 4), dims=[48, 48], compress=[1, 1],
            Cf=32, sp1=(8, 8, 8), classes=2, attractors=16, modes=4, qk_bias=True, ref_gflop=0.0, precision="tf32")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _grads_and_step(net, c, feat, curr, G, bench, milestones):
    from segtran_b200.parallel import GradBucket
    from segtran_b200.train import FlatBertAdam
    hp = bench.hot_params(net, c)
    bucket = GradBucket(hp, direct_accumulate=True, milestones=milestones)
    opt = FlatBertAdam([{"params": hp, "lr": 1e-3, "weight_decay": 1e-4}], warmup=-1, t_total=-1, grad_clip=0.1,
                       bucket=bucket)
    bucket.zero()
    f = feat.clone().requires_grad_()
    cc = curr.clone().requires_grad_()
    logits = net.hot_path(f, cc, None, (c["S"],) * 3)
    ((logits * G).sum() / feat.shape[0]).backward()
    bucket.allreduce_async()
    bucket.wait()
    grads = bucket.flat.clone()
    opt.step()
    torch.cuda.synchronize()
    return grads, hp, bucket


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    try:
        _worker_body(rank, dev, dist, q)
    except Exception:                                        # report instead of leaving the peer stuck in a collective
        import traceback
        q.put((rank, "error", traceback.format_exc()[-1500:], False))
    torch.cuda.synchronize()
    q.close()
    q.join_thread()
    os._exit(0)                                              # (no collective teardown: it can block on in-flight NCCL state)


def _worker_body(rank, dev, dist, q):
    if True:
        import bench
        import segtran_b200.networks.segtran_shared as S
        from segtran_b200 import ops
        S.bb2feat_dims["i3d"] = [8, 16, 24, 32, 48]      # (this subprocess only) tiny widths under the i3d shell
        c = TINY
        Bg = 4                                               # global batch, split 2 + 2
        g = torch.Generator().manual_seed(7)
        feat = torch.randn(Bg, c["dims"][0], *c["grid"], generator=g).to(dev)
        curr = torch.randn(Bg, c["Cf"], *c["sp1"], generator=g).to(dev)
        G = torch.randn(Bg, c["classes"], 16, 16, 16, generator=g).to(dev)
        lo, hi = rank * 2, rank * 2 + 2
        net = bench.build_net(c, "cuda", dropout=0.0).to(dev).train()
        grads, hp, bucket = _grads_and_step(net, c, feat[lo:hi], curr[lo:hi], G[lo:hi], bench, milestones=True)
        early = sum(bucket._sent)                            # every parameter went through a milestone or the final flush
        # parameters after the step: identical bits on every rank
        cs = bench.bucket_checksum(hp)
        mn, mx = cs.clone(), cs.clone()
        dist.all_reduce(mn, op=dist.ReduceOp.MIN)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        same_params = bool(torch.equal(mn, mx))
        # single-GPU reference on the concatenated batch (no process group involved: world-size-1 bucket semantics)
        ops.set_grad_ready_callback(None)
        ref = bench.build_net(c, "cuda", dropout=0.0).to(dev).train()
        hp_ref = bench.hot_params(ref, c)
        flat = torch.zeros(bucket.numel, device=dev)         # plain local gradient buffer in the bucket's layout
        for p, off in zip(hp_ref_unique(hp_ref), bucket.offsets):
            p.grad = flat[off:off + p.numel()].view_as(p)
        logits = ref.hot_path(feat.clone().requires_grad_(), curr.clone().requires_grad_(), None, (16, 16, 16))
        ((logits * G).sum() / Bg).backward()
        torch.cuda.synchronize()
        err = float((grads - flat).abs().max() / flat.abs().max())
        q.put((rank, same_params, err, early == len(bucket.params)))


def hp_ref_unique(ps):
    seen, out = set(), []
    for p in ps:
        if p.requires_grad and id(p) not in seen:
            seen.add(id(p))
            out.append(p)
    return out


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpu_dp_step_matches_single_gpu_and_ranks_agree():
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = []
    for _ in ps:
        res.append(q.get(timeout=240))
        if res[-1][1] == "error":
            for p in ps:
                p.kill()
            raise AssertionError("rank %d failed:\n%s" % (res[-1][0], res[-1][2]))
    for p in ps:
        p.join(timeout=60)
    print("2-GPU DP:", res)
    for rank, same_params, err, all_sent in res:
        assert same_params, "parameters differ between ranks after the update"
        assert err < 2e-3, "averaged gradient deviates from the single-GPU gradient of the full batch: %.2e" % err
        assert all_sent
