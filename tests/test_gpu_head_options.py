"""GPU checks of the head options --upd conv (folded into the collapsed head) and --outdrop (the dropout head of
csrc/sx_head_drop.cu): the shells against the reference fixtures, the kernels against the float64 oracle fed the
regenerated mask, determinism, CUDA-graph replay, class chunking and the memory the dropout head allocates."""
from argparse import Namespace

import pytest
import torch

from oracle import head_oracle as HO
from tests.helpers import load_golden, rel_err

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-3
GRAD_TOL = 5e-3
NAMES = ["seg3d_updconv", "seg3d_outdrop", "seg3d_updconv_outdrop", "seg2d_outdrop"]


class FixedFeat3d(torch.nn.Module):
    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def extract_features(self, x):
        keys = ["MaxPool3d_2a_3x3", "Conv3d_2c_3x3", "Mixed_3c", "Mixed_4f", "Mixed_5c"]
        return dict(zip(keys, self.feats))


class FixedFeat2d(torch.nn.Module):
    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def ext_features(self, x):
        return tuple(self.feats)


@pytest.fixture(params=["tf32", "tf32x3"])
def precision(request):
    from segtran_b200 import ops
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


def _build(name):
    import segtran_b200.networks.segtran_shared as S
    fx = load_golden(name)
    args = Namespace(**fx["args"])
    args.device = "cuda"
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    feats = [f.cuda().requires_grad_(i > 0) for i, f in enumerate(fx["feats"])]
    if fx["kind"] == "seg3d":
        import segtran_b200.networks.segtran3d as M
        cfg = M.Segtran3dConfig()
        cfg.update_config(args)
        net = M.Segtran3d(cfg, backbone=FixedFeat3d(feats))
    else:
        import segtran_b200.networks.segtran2d as M
        cfg = M.Segtran2dConfig()
        cfg.update_config(args)
        net = M.Segtran2d(cfg, backbone=FixedFeat2d(feats))
    net.load_state_dict(fx["state_dict"], strict=False)
    net = net.cuda()
    net.train() if fx["train"] else net.eval()
    return fx, net, feats


@pytest.mark.parametrize("name", NAMES)
def test_shell_matches_reference_fixture(name, precision):
    fx, net, feats = _build(name)
    y = net(fx["batch"].cuda())
    assert y.shape == fx["out"].shape
    e = rel_err(y, fx["out"])
    print(name, precision, "logits rel", e)
    assert e < OUT_TOL
    (y * fx["G"].cuda()).sum().backward()
    for i in range(1, 5):
        assert rel_err(feats[i].grad, fx["grad_feats"][i]) < GRAD_TOL, i
    gscale = max(float(g.abs().max()) for g in fx["grad_params"].values())
    got = dict(net.named_parameters())
    for k, g in fx["grad_params"].items():
        if k.startswith("backbone."):
            continue
        gg = got[k].grad
        if float(g.abs().max()) == 0.0:
            assert gg is None or float(gg.abs().max()) <= 1e-5 * gscale, k
            continue
        assert gg is not None, k
        err = float((gg.cpu() - g).abs().max())
        assert err <= GRAD_TOL * float(g.abs().max()) + 2e-5 * gscale, (k, err, float(g.abs().max()))


def _case(kind, upd="interp", B=2, Cf=16, Fd=32, K=3, Dk=2, sp=(6, 8, 12), grid=(3, 2, 3), seed=5):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)                     # noqa: E731
    if kind == 2:
        sp, grid = sp[1:], grid[1:]
    curr = r(B, Cf, *sp)
    vf = r(B, grid[0] * grid[1] * (grid[2] if len(grid) == 3 else 1), Fd)
    ones = (1,) * len(sp)
    Wb, bb = r(Fd, Cf, *ones) * 0.3, r(Fd)
    Fo = Fd // Dk if upd == "conv" else Fd
    Wc, bc = r(K, Fo, *ones) * 0.3, r(K)
    Wu, bu = (r(Fo * Dk, Fd, *ones) * 0.3, r(Fo * Dk)) if upd == "conv" else (None, None)
    return dict(curr=curr, vf=vf, Wb=Wb, bb=bb, Wc=Wc, bc=bc, Wu=Wu, bu=bu, grid=grid, Dk=Dk, Fo=Fo)


def _run(c, kind, upd, p, seed, out_size):
    from segtran_b200 import ops
    t = {k: (v.cuda().requires_grad_() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}
    y = ops.seg_head_dropout(t["curr"], t["vf"], c["grid"], t["Wb"], t["bb"], t["Wc"], t["bc"], out_size, p,
                             d_pool_k=c["Dk"], upsample_d=upd, Wu=t["Wu"], bu=t["bu"], seed=seed)
    return y, t


def _oracle(c, kind, upd, p, seed, out_size):
    t = {k: (v.double().requires_grad_() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}
    B = c["curr"].shape[0]
    vmap = t["vf"].transpose(1, 2).reshape(B, -1, *c["grid"])
    sp = c["curr"].shape[2:]
    if kind == 3:
        Dp = sp[0] * c["Dk"] if upd in ("interp", "conv") and c["Dk"] > 1 else sp[0]
        keep = HO.keep_mask(seed, (B, c["Fo"], Dp, sp[1], sp[2]), p)
        y = HO.seg_head_3d(t["curr"], vmap, t["Wb"], t["bb"], t["Wc"], t["bc"], out_size, c["Dk"], upd, t["Wu"],
                           t["bu"], keep=keep, p=p)
    else:
        keep = HO.keep_mask(seed, (B, c["Fo"], *sp), p)
        y = HO.seg_head_2d(t["curr"], vmap, t["Wb"], t["bb"], t["Wc"], t["bc"], out_size, keep=keep, p=p)
    return y, t


@pytest.mark.parametrize("kind,upd", [(3, "interp"), (3, "conv"), (3, "none"), (2, "none")])
def test_dropout_head_matches_oracle_with_regenerated_mask(kind, upd):
    from segtran_b200 import ops
    ops.set_precision("tf32x3")
    try:
        c = _case(kind, upd)
        out_size = (16, 24, 12) if kind == 3 else (16, 24)
        seed = 987654321
        y, t = _run(c, kind, upd, 0.3, seed, out_size)
        ref, tr = _oracle(c, kind, upd, 0.3, seed, out_size)
        assert rel_err(y, ref) < 1e-4
        G = torch.randn(ref.shape, dtype=torch.float64)
        (y * G.float().cuda()).sum().backward()
        (ref * G).sum().backward()
        for k in ("curr", "vf", "Wb", "bb", "Wc", "bc", "Wu", "bu"):
            if t[k] is None:
                continue
            assert rel_err(t[k].grad, tr[k].grad) < 1e-4, k
    finally:
        ops.set_precision("tf32")


def test_dropout_mask_statistics():
    """Kernel forward with p = 0.4 on a map of ones and a class row of ones: per-voxel score = kept channels / (1-p)."""
    from segtran_b200 import ops
    from segtran_b200 import _lib as L
    B, Fo, Ds, HW, p = 2, 256, 4, 1024, 0.4
    src = torch.ones(B, Fo, Ds, HW, device="cuda")
    Wc = torch.ones(1, Fo, device="cuda")
    Ls = ops._HeadDropout.apply(src, Wc, None, p, 4242, L.SX_HEAD_DMAP_NONE, 1)
    kept = Ls * (1 - p)
    frac = float(kept.mean()) / Fo
    assert abs(frac - (1 - p)) < 0.005
    # independent across voxels: the per-voxel count has the binomial variance
    var = float(kept.var())
    assert abs(var / (Fo * p * (1 - p)) - 1) < 0.1
    assert torch.allclose(kept, kept.round(), atol=1e-3)


def test_same_seed_same_bits_and_seeds_differ():
    c = _case(3, "interp")
    out = (16, 24, 12)
    ya, ta = _run(c, 3, "interp", 0.3, 11, out)
    ya.sum().backward()
    yb, tb = _run(c, 3, "interp", 0.3, 11, out)
    yb.sum().backward()
    yc, _ = _run(c, 3, "interp", 0.3, 12, out)
    assert torch.equal(ya, yb)
    for k in ("curr", "vf", "Wb", "Wc", "bc"):
        assert torch.equal(ta[k].grad, tb[k].grad), k
    assert not torch.equal(ya, yc)


def test_cuda_graph_replay_uses_device_seed():
    from segtran_b200 import ops
    c = _case(3, "interp")
    out = (16, 24, 12)
    t = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}
    seed_dev = torch.zeros(1, dtype=torch.int64, device="cuda")

    def step():
        return ops.seg_head_dropout(t["curr"], t["vf"], c["grid"], t["Wb"], t["bb"], t["Wc"], t["bc"], out, 0.3,
                                    d_pool_k=2, seed=seed_dev)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = step()
    outs = []
    for sv in (101, 202):
        seed_dev.fill_(sv)
        g.replay()
        torch.cuda.synchronize()
        outs.append(y.clone())
        eager = ops.seg_head_dropout(t["curr"], t["vf"], c["grid"], t["Wb"], t["bb"], t["Wc"], t["bc"], out, 0.3,
                                     d_pool_k=2, seed=sv)
        assert torch.equal(outs[-1], eager)
    assert not torch.equal(outs[0], outs[1])


def test_more_than_eight_folded_classes_run_in_chunks():
    """--upd conv with K * D_pool_K = 5 * 2 = 10 class rows: the collapsed head runs two chunks; and the dropout head
    with K = 9 classes runs its class chunks."""
    from segtran_b200 import ops
    ops.set_precision("tf32x3")
    try:
        c = _case(3, "conv", K=5)
        out = (16, 24, 12)
        t = {k: (v.cuda().requires_grad_() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}
        Wf, bf = ops.fold_unfold(t["Wc"], t["bc"], t["Wu"], t["bu"], 2)
        y = ops.seg_head(t["curr"], t["vf"], c["grid"], t["Wb"], t["bb"], Wf, bf, out, d_unfold=2)
        ref, tr = _oracle(c, 3, "conv", 0.0, 0, out)
        assert rel_err(y, ref) < 1e-4
        G = torch.randn(ref.shape, dtype=torch.float64)
        (y * G.float().cuda()).sum().backward()
        (ref * G).sum().backward()
        for k in ("curr", "vf", "Wb", "bb", "Wc", "bc", "Wu", "bu"):
            assert rel_err(t[k].grad, tr[k].grad) < 1e-4, k
        c9 = _case(3, "interp", K=9)
        y9, t9 = _run(c9, 3, "interp", 0.3, 77, out)
        r9, tr9 = _oracle(c9, 3, "interp", 0.3, 77, out)
        assert rel_err(y9, r9) < 1e-4
        G = torch.randn(r9.shape, dtype=torch.float64)
        (y9 * G.float().cuda()).sum().backward()
        (r9 * G).sum().backward()
        for k in ("curr", "Wc", "bc"):
            assert rel_err(t9[k].grad, tr9[k].grad) < 1e-4, k
    finally:
        ops.set_precision("tf32")


def test_dropout_head_never_allocates_the_dropped_map():
    """interp x4 on a [1,256,16,64,64] source: the dropped map X would be 4x the source (256 MB).  The kernels'
    forward + backward allocate the scores, their gradient and dsrc (the source's size), nothing of X's size."""
    from segtran_b200 import ops
    from segtran_b200 import _lib as L
    B, Fo, Ds, HW, Dk, K = 1, 256, 16, 64 * 64, 4, 3
    src = torch.randn(B, Fo, Ds, HW, device="cuda", requires_grad=True)
    Wc = torch.randn(K, Fo, device="cuda", requires_grad=True)
    bc = torch.randn(K, device="cuda", requires_grad=True)
    x_bytes = B * Fo * Ds * Dk * HW * 4
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    Ls = ops._HeadDropout.apply(src, Wc, bc, 0.2, 5, L.SX_HEAD_DMAP_INTERP, Dk)
    Ls.backward(torch.ones_like(Ls))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("peak extra MB", peak / 2 ** 20, "dropped map MB", x_bytes / 2 ** 20)
    assert peak < 0.4 * x_bytes
