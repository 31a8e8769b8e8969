"""GPU checks of the 2.5-D model: the cross-slice GroupNorm kernels (sx_groupnorm_slices_fwd/bwd through
ops.group_norm(slices=D)) against float64 nn.GroupNorm on the stacked [B,C,h,w,D] volume, and the Segtran25d shell
against the reference fixtures (tests/golden/seg25d_*.pt, built from the real reference by
oracle/gen_seg25d_golden.py): logits, gradients to the parameters and features, masks, and run-to-run determinism."""
from argparse import Namespace

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import load_golden, rel_err

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-3
GRAD_TOL = 5e-3
NAMES = ["seg25d_stemconv", "seg25d_updconv", "seg25d_dgroup2", "seg25d_direct34", "seg25d_posbias"]


# (B, D, C, G, spatial): D = 1 (the plain GroupNorm), 3 and 8 slices; V % 4 != 0 (generic path); G = C; the eff-b3
# out-FPN level at the full shape; more than 65535 (b, d, c) rows
GN_CASES = [
    (2, 1, 16, 8, (8, 8)),
    (2, 3, 16, 8, (8, 8)),
    (2, 8, 24, 8, (5, 7)),
    (3, 3, 12, 12, (4, 4)),
    (1, 96, 48, 8, (56, 56)),
    (2, 96, 384, 8, (2, 2)),
]


@pytest.mark.parametrize("B,D,C,G,sp", GN_CASES)
@pytest.mark.parametrize("offset", [0, 1])
def test_slice_group_norm_matches_float64_volume(B, D, C, G, sp, offset):
    from segtran_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + D * 10 + C + offset)
    n = B * D * C * sp[0] * sp[1]
    buf = torch.randn(n + offset, generator=g) * 2.0 + 0.5
    x = buf[offset:].view(B * D, C, *sp)                 # offset 1: a 4-byte-aligned view, the generic (scalar) path
    gamma = torch.randn(C, generator=g)
    beta = torch.randn(C, generator=g)
    dy = torch.randn(B * D, C, *sp, generator=g)

    def vol(t):                                          # [B*D, C, h, w] -> [B, C, h, w, D]
        return t.reshape(B, D, C, *sp).permute(0, 2, 3, 4, 1)

    xr, gr, br = (t.double().requires_grad_() for t in (x, gamma, beta))
    yr = F.group_norm(vol(xr), G, gr, br, 1e-5)
    yr.backward(vol(dy.double()))

    xb = buf.cuda()[offset:].view(B * D, C, *sp).requires_grad_()
    gb, bb = gamma.cuda().requires_grad_(), beta.cuda().requires_grad_()
    yb = ops.group_norm(xb, gb, bb, G, 1e-5, slices=D)
    yb.backward(dy.cuda())
    assert rel_err(vol(yb), yr) < 1e-5
    assert rel_err(xb.grad, xr.grad) < 1e-4
    assert rel_err(gb.grad, gr.grad) < 1e-4
    assert rel_err(bb.grad, br.grad) < 1e-4


class FixedFeat(torch.nn.Module):
    """The stored per-slice feature maps, as either backbone's feature call returns them."""

    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def ext_features(self, x):
        assert x.shape[0] == self.feats[1].shape[0]
        return tuple(self.feats)

    def extract_endpoints(self, x):
        return {'reduction_%d' % (i + 1): f for i, f in enumerate(self.ext_features(x))}


def _build(name):
    import segtran_b200.networks.segtran_shared as S
    import segtran_b200.networks.segtran25d as M
    fx = load_golden(name)
    args = Namespace(**fx["args"])
    args.device = "cuda"
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    feats = [f.cuda().requires_grad_(i > 0) for i, f in enumerate(fx["feats"])]
    cfg = M.Segtran25dConfig()
    cfg.update_config(args)
    cfg.max_pos_size = tuple(fx["grid"])
    net = M.Segtran25d(cfg, backbone=FixedFeat(feats))
    net.load_state_dict(fx["state_dict"], strict=True)
    net = net.cuda().eval()
    return fx, net, feats


@pytest.mark.parametrize("name", NAMES)
def test_shell_matches_reference_fixture(name):
    fx, net, feats = _build(name)
    y = net(fx["batch"].cuda())
    assert y.shape == fx["out"].shape
    e = rel_err(y, fx["out"])
    print(name, "logits rel", e)
    assert e < OUT_TOL
    (y * fx["G"].cuda()).sum().backward()
    for i in range(1, 5):
        if fx["grad_feats"][i] is None:
            assert feats[i].grad is None or float(feats[i].grad.abs().max()) == 0.0, i
            continue
        assert rel_err(feats[i].grad, fx["grad_feats"][i]) < GRAD_TOL, i
    gscale = max(float(g.abs().max()) for g in fx["grad_params"].values())
    got = dict(net.named_parameters())
    for k, g in fx["grad_params"].items():
        gg = got[k].grad
        if float(g.abs().max()) == 0.0:
            assert gg is None or float(gg.abs().max()) <= 1e-5 * gscale, k
            continue
        assert gg is not None, k
        err = float((gg.cpu() - g).abs().max())
        assert err <= GRAD_TOL * float(g.abs().max()) + 2e-5 * gscale, (k, err, float(g.abs().max()))


@pytest.mark.parametrize("name", ["seg25d_stemconv", "seg25d_updconv"])
def test_hard_masks_match_reference(name):
    fx, net, _ = _build(name)
    with torch.no_grad():
        y = net(fx["batch"].cuda()).cpu()
    ref = fx["out"]
    top2 = ref.topk(2, dim=1).values
    sure = (top2[:, 0] - top2[:, 1]) > 1e-4                   # argmax not within rounding of a tie
    assert torch.equal(y.argmax(1)[sure], ref.argmax(1)[sure])
    sure = (torch.sigmoid(ref) - 0.5).abs() > 1e-4
    assert torch.equal((torch.sigmoid(y) > 0.5)[sure], (torch.sigmoid(ref) > 0.5)[sure])


def test_runs_are_bit_identical():
    outs = []
    for _ in range(2):
        fx, net, feats = _build("seg25d_updconv")
        y = net(fx["batch"].cuda())
        (y * fx["G"].cuda()).sum().backward()
        outs.append([y.detach().clone()] + [f.grad.clone() for f in feats[1:]] +
                    [p.grad.clone() for p in net.parameters() if p.grad is not None])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_cuda_graph_replay_of_forward_loss_backward():
    """Forward + loss + backward of the shell captured once (segtran_b200/graph.py) and replayed: same logits and
    gradients as the reference fixture, and two replays are bit-identical."""
    from segtran_b200.graph import CapturedStep
    fx, net, feats = _build("seg25d_updconv")
    net.train()                                                   # dropout 0 in the fixture
    batch, G = fx["batch"].cuda(), fx["G"].cuda()

    def step():
        for f in feats[1:]:
            f.grad = None
        for p_ in net.parameters():
            p_.grad = None
        y = net(batch)
        (y * G).sum().backward()
        return y

    g = CapturedStep(step, warmup=2)
    y1 = g().clone()
    gr1 = [f.grad.clone() for f in feats[1:]]
    y2 = g().clone()
    assert torch.equal(y1, y2)
    assert all(torch.equal(a, f.grad) for a, f in zip(gr1, feats[1:]))
    assert rel_err(y1, fx["out"]) < OUT_TOL
    for i in range(1, 5):
        assert rel_err(feats[i].grad, fx["grad_feats"][i]) < GRAD_TOL, i
    assert g.kernel_launches > 20


class _Replay(torch.nn.Module):
    """Returns stored logits (cut to the input's batch) on the input's device: the oracle's stand-in for the net."""

    def __init__(self, y):
        super().__init__()
        self.y = y

    def forward(self, x):
        return self.y[:x.shape[0]].to(x.device)


def test_sliding_window_inference_on_a_25d_net():
    from oracle import infer_oracle as IO
    from segtran_b200.inference import test_single_case
    fx, net, _ = _build("seg25d_updconv")                         # bridgeconv: every slice is unmasked
    image = torch.randn(2, 16, 16, 16, generator=torch.Generator().manual_seed(2))
    windows = torch.stack([image[..., 0:8], image[..., 8:16]])    # the two windows along D, in visiting order
    with torch.no_grad():
        y = net(windows.cuda()).cpu()
    args = ((16, 16, 8), (16, 16, 8), 2, 8, 8, "atria", "segtran", 3)
    hard, soft = test_single_case(net, image.cuda(), *args)
    ref_hard, ref_soft = IO.test_single_case(_Replay(y), image, *args)
    assert soft.shape == ref_soft.shape == (3, 16, 16, 16)
    assert float((soft.cpu() - ref_soft).abs().max()) < 1e-5
    top2 = ref_soft.topk(2, dim=0).values
    sure = (top2[0] - top2[1]) > 1e-4
    assert torch.equal(hard.cpu()[sure], ref_hard[sure])


def build_fullsize(B=1, seed=0):
    """The real shape: input [B,4,112,112,96], eff-b3 feature widths, --infpn 34 --outfpn 1234, stemconv, --upd conv,
    1024 attractors: token grid (14,14,48) = 9408 tokens x 1536 channels, out-FPN head 56x56 on 96 slices.  The backbone
    is a stand-in returning seeded per-slice features; the first 8 depth slices of the input are empty (masked)."""
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


def test_fullsize_matches_oracle_on_gpu():
    from oracle import seg25d_oracle as SO
    cfg, net, feats, batch = build_fullsize()
    assert net.trans_in_dim == 1536 and cfg.num_attractors == 1024
    with torch.no_grad():
        y = net(batch)
        assert net.orig_feat_shape == (14, 14, 48)
        p = {k: v for k, v in net.state_dict().items()}
        old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        try:
            ref = SO.forward(p, feats, SO.get_mask(batch, 8), 1, (112, 112, 96), in_layers=net.in_fpn_layers,
                             out_layers=net.out_fpn_layers, translayer_dims=net.translayer_dims,
                             num_modes=cfg.num_modes, D_pool_K=2, upd='conv')
        finally:
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    assert y.shape == ref.shape == (1, 2, 112, 112, 96)
    e = rel_err(y, ref)
    print("full-size logits rel", e)
    assert e < OUT_TOL
