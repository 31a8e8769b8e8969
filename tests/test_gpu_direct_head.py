"""GPU checks of the class head without the out-FPN (out_fpn_layers == in_fpn_layers; ops.direct_head, the widened
sx_token_scores and sx_subpixel_resize_fwd/bwd): the kernels against the float64 oracle in 2-D and 3-D, the shells
against the reference fixtures, determinism, CUDA-graph replay, and sliding-window inference on a direct-head net."""
from argparse import Namespace

import pytest
import torch

from oracle import direct_head_oracle as DO
from oracle import eval2d_oracle as E
from oracle import infer_oracle as IO
from tests.helpers import load_golden, rel_err

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-3
GRAD_TOL = 5e-3
NAMES = ["seg2d_direct34", "seg2d_direct234", "seg3d_direct34", "seg3d_direct34_outdrop"]


class FixedFeat3d(torch.nn.Module):
    """The stored feature maps, cut to the batch of the input (at most the fixture's)."""

    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def extract_features(self, x):
        keys = ["MaxPool3d_2a_3x3", "Conv3d_2c_3x3", "Mixed_3c", "Mixed_4f", "Mixed_5c"]
        return dict(zip(keys, [f[:x.shape[0]] for f in self.feats]))


class FixedFeat2d(torch.nn.Module):
    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def ext_features(self, x):
        return tuple(f[:x.shape[0]] for f in self.feats)


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
        if fx["grad_feats"][i] is None:                      # levels that only the out-FPN reads
            assert feats[i].grad is None, i
            continue
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


def _case(K, grid, C, B=2, seed=7):
    g = torch.Generator().manual_seed(seed)
    N = 1
    for v in grid:
        N *= v
    x = torch.randn(B, N, C, generator=g)
    Wt = torch.randn(C, K, 2, 2, *((1,) if len(grid) == 3 else ()), generator=g) * 0.2
    bt = torch.randn(K, generator=g)
    return x, Wt, bt


def _oracle(x, Wt, bt, grid, out_size):
    B, N, C = x.shape
    return DO.direct_head(x.transpose(1, 2).reshape(B, C, *grid), Wt, bt, out_size)


# (K, token grid, channels, output size): 2-D grids (H2,W2) -> (H,W); 3-D grids (D2,H2,W2) -> (H,W,D).  Odd grids, odd
# token counts (the CUDA-core dW path), C % 4 != 0 (the CUDA-core dX path), up- and down-sampling, sizes that are not
# multiples of the sub-pixel grid, and 4, 8, 12, 16 and 32 sub-pixel rows
CASES = [
    (1, (7, 5), 16, (20, 13)),
    (2, (6, 8), 32, (24, 32)),
    (3, (5, 6), 30, (11, 40)),
    (8, (4, 4), 20, (16, 16)),
    (1, (3, 7, 5), 16, (20, 13, 9)),
    (2, (2, 3, 4), 22, (12, 16, 5)),
    (3, (3, 4, 4), 24, (16, 16, 24)),
    (4, (3, 7, 5), 18, (28, 20, 7)),
    (8, (2, 3, 2), 12, (9, 8, 6)),
]


@pytest.mark.parametrize("K,grid,C,out_size", CASES)
def test_kernels_match_float64_oracle(K, grid, C, out_size):
    from segtran_b200 import ops
    ops.set_precision("tf32x3")                         # the dW product is a tensor-core GEMM: 3 passes for fp32 grade
    try:
        x, Wt, bt = _case(K, grid, C)
        t = [v.cuda().requires_grad_() for v in (x, Wt, bt)]
        y = ops.direct_head(t[0], grid, t[1], t[2], out_size)
        r = [v.double().requires_grad_() for v in (x, Wt, bt)]
        ref = _oracle(*r, grid, out_size)
        assert y.shape == ref.shape
        e = rel_err(y, ref)
        G = torch.randn(ref.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
        (y * G.float().cuda()).sum().backward()
        (ref * G.float().double()).sum().backward()
        errs = [rel_err(a.grad, b.grad) for a, b in zip(t, r)]
        print(K, grid, C, out_size, "logits", e, "dX dW db", errs)
        assert e < 1e-5
        assert errs[0] < 1e-5 and errs[2] < 1e-5
        assert errs[1] < 1e-4
    finally:
        ops.set_precision("tf32")


def test_no_bias():
    from segtran_b200 import ops
    x, Wt, _ = _case(2, (3, 4, 4), 16)
    y = ops.direct_head(x.cuda(), (3, 4, 4), Wt.cuda(), None, (12, 16, 9))
    assert rel_err(y, _oracle(x, Wt, None, (3, 4, 4), (12, 16, 9))) < 1e-5


def _fwd_bwd(t, grid, out_size, G):
    from segtran_b200 import ops
    y = ops.direct_head(t[0], grid, t[1], t[2], out_size)
    return (y,) + torch.autograd.grad(y, t, G)


@pytest.mark.parametrize("grid,out_size", [((14, 14, 14), (112, 112, 112)), ((36, 36), (288, 288))])
def test_two_runs_give_the_same_bits(grid, out_size):
    x, Wt, bt = _case(4 if len(grid) == 3 else 3, grid, 64, B=2)
    t = [v.cuda().requires_grad_() for v in (x, Wt, bt)]
    G = torch.randn((2, Wt.shape[1]) + out_size, device="cuda")
    a = _fwd_bwd(t, grid, out_size, G)
    b = _fwd_bwd(t, grid, out_size, G)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_cuda_graph_replay_equals_eager():
    grid, out_size = (3, 7, 5), (28, 20, 12)
    x, Wt, bt = _case(4, grid, 32)
    t = [v.cuda().requires_grad_() for v in (x, Wt, bt)]
    G = torch.randn((2, 4) + out_size, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _fwd_bwd(t, grid, out_size, G)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        outs = _fwd_bwd(t, grid, out_size, G)
    with torch.no_grad():
        t[0].mul_(0.5)
        G.mul_(-2.0)
    g.replay()
    torch.cuda.synchronize()
    eager = _fwd_bwd(t, grid, out_size, G)
    for u, v in zip(outs, eager):
        assert torch.equal(u, v)


class _Replay(torch.nn.Module):
    """Returns stored logits (cut to the input's batch) on the input's device: the oracle's stand-in for the net."""

    def __init__(self, y):
        super().__init__()
        self.y = y

    def forward(self, x):
        return self.y[:x.shape[0]].to(x.device)


def test_sliding_window_inference_3d_on_a_direct_head_net():
    from segtran_b200.inference import test_single_case
    fx, net, _ = _build("seg3d_direct34")
    with torch.no_grad():
        y = net(fx["batch"].cuda()).cpu()
    image = torch.randn(4, 16, 16, 32, generator=torch.Generator().manual_seed(2))
    args = ((16, 16, 24), (16, 16, 24), 2, 8, 8, "atria", "segtran", 3)       # two windows along D, one batch
    hard, soft = test_single_case(net, image.cuda(), *args)
    ref_hard, ref_soft = IO.test_single_case(_Replay(y), image, *args)
    assert soft.shape == ref_soft.shape == (3, 16, 16, 32)
    assert float((soft.cpu() - ref_soft).abs().max()) < 1e-5
    top2 = ref_soft.topk(2, dim=0).values
    sure = (top2[0] - top2[1]) > 1e-4
    assert torch.equal(hard.cpu()[sure], ref_hard[sure])


def test_sliding_window_inference_2d_on_a_direct_head_net():
    from segtran_b200.inference import test_single_batch
    fx, net, _ = _build("seg2d_direct34")
    with torch.no_grad():
        y = net(fx["batch"].cuda()).cpu()
    image = torch.randn(2, 3, 32, 48, generator=torch.Generator().manual_seed(3))
    args = ((32, 32), (32, 32), (16, 16), "fundus", 3, "segtran")              # two windows along W
    hard, soft = test_single_batch(net, image.cuda(), *args)
    ref_hard, ref_soft = E.test_single_batch(_Replay(y), image, *args)
    assert soft.shape == tuple(ref_soft.shape) == (2, 3, 32, 48)
    assert float((soft.cpu() - torch.as_tensor(ref_soft)).abs().max()) < 1e-5
