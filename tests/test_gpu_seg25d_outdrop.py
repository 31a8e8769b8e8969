"""GPU checks of the 2.5-D --outdrop head (ops.seg_head_slices_dropout: csrc/sx_head_drop.cu reading the slice-major
map, with the interleaved depth unfold for --upd conv): the Segtran25d shell in training against the reference fixtures
(tests/golden/seg25d_outdrop_*.pt), the op against the float64 oracle fed the regenerated mask, the mask's statistics,
determinism, CUDA-graph replay, and the full 2.5-D shape (memory and accuracy)."""
from argparse import Namespace

import pytest
import torch

from oracle import head_oracle as HO
from oracle import seg25d_outdrop_oracle as DO
from segtran_b200 import _lib as L
from tests.helpers import load_golden, rel_err

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-3
GRAD_TOL = 5e-3
NAMES = ["seg25d_outdrop_updconv", "seg25d_outdrop_interp", "seg25d_outdrop_noupd", "seg25d_outdrop_dk1",
         "seg25d_outdrop_k5"]


class FixedFeat(torch.nn.Module):
    def __init__(self, feats):
        super().__init__()
        self.feats = feats

    def ext_features(self, x):
        return tuple(self.feats)

    def extract_endpoints(self, x):
        return {'reduction_%d' % (i + 1): f for i, f in enumerate(self.feats)}


@pytest.fixture(params=["tf32", "tf32x3"])
def precision(request):
    from segtran_b200 import ops
    old = ops.get_precision()
    ops.set_precision(request.param)
    yield request.param
    ops.set_precision(old)


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
    return fx, net.cuda().train(), feats


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
        gg = got[k].grad
        if float(g.abs().max()) == 0.0:
            assert gg is None or float(gg.abs().max()) <= 1e-5 * gscale, k
            continue
        assert gg is not None, k
        err = float((gg.cpu() - g).abs().max())
        assert err <= GRAD_TOL * float(g.abs().max()) + 2e-5 * gscale, (k, err, float(g.abs().max()))


def _case(upd, Dk=2, B=2, D2=4, Cf=12, Fd=16, H1=6, W1=8, grid=(3, 2, 2), K=3, seed=5):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)                     # noqa: E731
    conv = upd == "conv" and Dk > 1
    Fo = Fd // Dk if conv else Fd
    return dict(curr=r(B * D2, Cf, H1, W1), vf=r(B, grid[0] * grid[1] * grid[2], Fd), Wb=r(Fd, Cf, 1, 1, 1) * 0.3,
                bb=r(Fd), Wc=r(K, Fo, 1, 1, 1) * 0.3, bc=r(K), Wu=r(Fo * Dk, Fd, 1, 1, 1) * 0.3 if conv else None,
                bu=r(Fo * Dk) if conv else None, grid=grid, Dk=Dk, Fo=Fo, B=B, D2=D2, upd=upd)


def _run(c, p, seed, out_size):
    from segtran_b200 import ops
    t = {k: (v.cuda().requires_grad_() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}
    y = ops.seg_head_slices_dropout(t["curr"], t["vf"], c["grid"], t["Wb"], t["bb"], t["Wc"], t["bc"], out_size, p,
                                    c["Dk"], c["upd"], Wu=t["Wu"], bu=t["bu"], seed=seed)
    return y, t


def _depth_out(c):
    return c["D2"] * c["Dk"] if c["upd"] in ("conv", "interpolate") and c["Dk"] > 1 else c["D2"]


def _oracle(c, p, seed, out_size, device="cpu"):
    t = {k: (v.to(device).double().requires_grad_() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}
    H1, W1 = c["curr"].shape[2:]
    keep = DO.keep_mask_torch(seed, (c["B"], c["Fo"], _depth_out(c), H1, W1), p, device)
    y = DO.head_25d(t["curr"], t["vf"], c["grid"], t["Wb"], t["bb"], t["Wc"], t["bc"], out_size, c["Dk"], c["upd"],
                    t["Wu"], t["bu"], keep=keep, p=p)
    return y, t


DMAP_CASES = [("conv", 2), ("interpolate", 2), ("interp", 2), ("none", 2), ("conv", 1), ("conv", 3)]


@pytest.mark.parametrize("upd,Dk", DMAP_CASES)
def test_dropout_head_matches_oracle_with_regenerated_mask(upd, Dk):
    from segtran_b200 import ops
    ops.set_precision("tf32x3")
    try:
        c = _case(upd, Dk=Dk, D2=6 if Dk == 3 else 4, grid=(3, 2, 2))
        out_size = (12, 16, c["D2"] * 2)
        seed = 987654321
        y, t = _run(c, 0.3, seed, out_size)
        ref, tr = _oracle(c, 0.3, seed, out_size)
        assert y.shape == ref.shape
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


def _kernel_ref(src, layout, Wc, bc, keep, p, dmap, Dk):
    """Float64 restatement of sx_head_dropout_fwd on a source of either layout -> Ls [B,K,D',HW]."""
    s = src.double()
    if layout == L.SX_HEAD_SRC_SLICE_MAJOR:
        s = s.transpose(1, 2)                                        # -> [B, Fs, Ds, HW]
    B, Fs, Ds, HW = s.shape
    if dmap == L.SX_HEAD_DMAP_INTERP:
        X = torch.nn.functional.interpolate(s, size=(Ds * Dk, HW), mode="bilinear", align_corners=False)
    elif dmap == L.SX_HEAD_DMAP_UNFOLD:                              # X[f, j Ds + i] = src[f Dk + j, i]
        X = s.reshape(B, Fs // Dk, Dk * Ds, HW)
    elif dmap == L.SX_HEAD_DMAP_UNFOLD_INTERLEAVED:                  # X[f, i Dk + j] = src[f Dk + j, i]
        X = s.reshape(B, Fs // Dk, Dk, Ds, HW).transpose(2, 3).reshape(B, Fs // Dk, Ds * Dk, HW)
    else:
        X = s
    X = X * keep.double() / (1.0 - p)
    return torch.einsum("kf,bfdv->bkdv", Wc.double(), X) + bc.double().view(1, -1, 1, 1)


@pytest.mark.parametrize("HW", [35, 48])
@pytest.mark.parametrize("dmap", [0, 1, 2, 3])
@pytest.mark.parametrize("layout", [0, 1])
def test_kernel_layouts_and_depth_maps_match_float64(layout, dmap, HW):
    """The kernels alone on either layout, every depth map; HW = 35 takes the scalar path, 48 the vector one."""
    from segtran_b200 import ops
    g = torch.Generator().manual_seed(layout * 100 + dmap * 10 + HW)
    B, Fs, Ds, K, p, seed = 2, 12, 5, 5, 0.3, 4321
    Dk = 3 if dmap in (L.SX_HEAD_DMAP_UNFOLD, L.SX_HEAD_DMAP_UNFOLD_INTERLEAVED) else (2 if dmap else 1)
    Fo = Fs // Dk if dmap in (L.SX_HEAD_DMAP_UNFOLD, L.SX_HEAD_DMAP_UNFOLD_INTERLEAVED) else Fs
    Do = Ds if dmap == L.SX_HEAD_DMAP_NONE else Ds * Dk
    shape = (B, Ds, Fs, HW) if layout == L.SX_HEAD_SRC_SLICE_MAJOR else (B, Fs, Ds, HW)
    src = torch.randn(*shape, generator=g)
    Wc, bc = torch.randn(K, Fo, generator=g), torch.randn(K, generator=g)
    keep = DO.keep_mask_torch(seed, (B, Fo, Do, HW), p, "cpu")
    s64, W64, b64 = (x.double().requires_grad_() for x in (src, Wc, bc))
    ref = _kernel_ref(s64, layout, W64, b64, keep, p, dmap, Dk)
    sg, Wg, bg = (x.cuda().requires_grad_() for x in (src, Wc, bc))
    Ls = ops._HeadDropout.apply(sg, Wg, bg, p, seed, dmap, Dk, layout)
    assert Ls.shape == ref.shape
    assert rel_err(Ls, ref) < 1e-5
    dL = torch.randn(ref.shape, generator=g)
    Ls.backward(dL.cuda())
    ref.backward(dL.double())
    for a, b in ((sg, s64), (Wg, W64), (bg, b64)):
        assert rel_err(a.grad, b.grad) < 1e-5


def test_mask_statistics_and_forward_backward_masks_agree():
    """Slice-major source of ones, Wc = identity (F' classes, so four class chunks): Ls[b,k,d,hw] = keep(b,k,d,hw)/(1-p).
    The keep rate is within binomial bounds, and with dLs = 1 the gradient dsrc[b,d,f,hw] = keep(b,f,d,hw)/(1-p): zero
    exactly where the forward dropped."""
    from segtran_b200 import ops
    B, Fo, Ds, HW, p = 2, 16, 8, 1024, 0.3
    src = torch.ones(B, Ds, Fo, HW, device="cuda", requires_grad=True)
    Wc = torch.eye(Fo, device="cuda")
    Ls = ops._HeadDropout.apply(src, Wc, None, p, 777, L.SX_HEAD_DMAP_NONE, 1, L.SX_HEAD_SRC_SLICE_MAJOR)
    fwd_keep = Ls != 0
    n = fwd_keep.numel()
    rate = float(fwd_keep.float().mean())
    sd = ((1 - p) * p / n) ** 0.5
    assert abs(rate - (1 - p)) < 5 * sd, (rate, sd)
    assert torch.allclose(Ls[fwd_keep], torch.full_like(Ls[fwd_keep], 1 / (1 - p)))
    Ls.backward(torch.ones_like(Ls))
    bwd_keep = (src.grad != 0).transpose(1, 2)                       # [B, F, Ds, HW]
    assert torch.equal(bwd_keep, fwd_keep)
    assert torch.equal(fwd_keep.cpu(), HO.keep_mask(777, (B, Fo, Ds, HW), p).bool())


def test_same_seed_same_bits_and_seeds_differ():
    c = _case("conv")
    out = (12, 16, 8)
    ya, ta = _run(c, 0.3, 11, out)
    ya.sum().backward()
    yb, tb = _run(c, 0.3, 11, out)
    yb.sum().backward()
    yc, _ = _run(c, 0.3, 12, out)
    assert torch.equal(ya, yb)
    for k in ("curr", "vf", "Wb", "bb", "Wc", "bc", "Wu", "bu"):
        assert torch.equal(ta[k].grad, tb[k].grad), k
    assert not torch.equal(ya, yc)


def test_captured_training_step_takes_a_new_mask_per_replay():
    """Segtran25d forward + loss + backward with --outdrop p = 0.3 captured as a CUDA graph: each replay after
    ops.advance_seed draws new per-call seeds on the device, and its logits and gradients equal those of an eager step
    given that replay's seeds."""
    from segtran_b200 import ops
    from segtran_b200.graph import CapturedStep
    fx, net, feats = _build("seg25d_outdrop_updconv")
    net.out_fpn_dropout.p = 0.3
    batch, G = fx["batch"].cuda(), fx["G"].cuda()
    seeds, given = [], []
    orig = ops.new_dropout_seed

    def recording(device):
        if given:
            return given.pop(0)
        t = orig(device)
        seeds.append(t)
        return t

    def step():
        for f in feats[1:]:
            f.grad = None
        for p_ in net.parameters():
            p_.grad = None
        seeds.clear()
        y = net(batch)
        (y * G).sum().backward()
        return y

    ops.new_dropout_seed = recording
    try:
        graph = CapturedStep(step, warmup=2)
        graph_seeds = list(seeds)
        graph_grads = [f.grad for f in feats[1:]] + [p_.grad for p_ in net.parameters()]
        assert graph_seeds
        outs = []
        for _ in range(2):
            ops.advance_seed(batch.device)
            y = graph().clone()
            torch.cuda.synchronize()
            grads = [g.clone() for g in graph_grads if g is not None]
            outs.append(y)
            given[:] = [s.clone() for s in graph_seeds]              # that replay's seeds, for the eager step
            ye = step()
            torch.cuda.synchronize()
            assert not given
            assert torch.equal(ye, y)
            eager = [f.grad for f in feats[1:]] + [p_.grad for p_ in net.parameters()]
            assert all(torch.equal(a, b) for a, b in zip(grads, [g for g in eager if g is not None]))
        assert not torch.equal(outs[0], outs[1])
        assert graph.kernel_launches > 20
    finally:
        ops.new_dropout_seed = orig


def _fullsize_head_inputs(upd, seed=0):
    """The full 2.5-D head: out-FPN map [96, 136, 56, 56] (eff-b3, input [1,4,112,112,96]), fused tokens on the
    (14, 14, 48) grid with 1536 channels, 2 classes, D_pool_K = 2."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)                     # noqa: E731
    B, D2, Cf, Fd, K, Dk, grid = 1, 96, 136, 1536, 2, 2, (14, 14, 48)
    conv = upd == "conv"
    Fo = Fd // Dk if conv else Fd
    return dict(curr=r(B * D2, Cf, 56, 56), vf=r(B, 14 * 14 * 48, Fd), Wb=r(Fd, Cf, 1, 1, 1) * 0.05, bb=r(Fd) * 0.1,
                Wc=r(K, Fo, 1, 1, 1) * 0.03, bc=r(K) * 0.1, Wu=r(Fo * Dk, Fd, 1, 1, 1) * 0.03 if conv else None,
                bu=r(Fo * Dk) * 0.1 if conv else None, grid=grid, Dk=Dk, Fo=Fo, B=B, D2=D2, upd=upd)


@pytest.mark.parametrize("upd", ["conv", "interpolate"])
def test_fullsize_memory_and_accuracy(upd, precision):
    """At the real shape the head holds the slice-major maps it must and never the dropped, depth-upsampled one:
    the bridge GEMM's output Y with its addend (the upsampled tokens, an input of the GEMM's epilogue); for --upd conv
    also Y's TF32 operand copy kept for the upsampleD GEMM's backward, and Y2; the class scores and the logits (checked
    in tf32, the training precision).
    Forward and backward match the float64 oracle fed the regenerated mask: logits and the gradients to the features
    and the class conv within 1e-3; the bridge and upsampleD weight gradients, each a conv1x1_add weight-gradient GEMM
    summed over 301k voxels in fp32, within the fixtures' 5e-3 (about 2e-3 in either precision on an H100)."""
    from segtran_b200 import ops
    c = _fullsize_head_inputs(upd)
    out_size, p, seed = (112, 112, 96), 0.2, 24680
    t = {k: (v.cuda().requires_grad_() if isinstance(v, torch.Tensor) else v) for k, v in c.items()}
    M = c["B"] * c["D2"] * 1536 * 56 * 56 * 4                        # one slice-major map
    Do = _depth_out(c)
    ls_bytes = c["B"] * 2 * Do * 56 * 56 * 4
    out_bytes = c["B"] * 2 * 112 * 112 * 96 * 4
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    y = ops.seg_head_slices_dropout(t["curr"], t["vf"], c["grid"], t["Wb"], t["bb"], t["Wc"], t["bc"], out_size, p,
                                    c["Dk"], upd, Wu=t["Wu"], bu=t["bu"], seed=seed)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    maps = 3 if upd == "conv" else 2
    budget = maps * M + ls_bytes + 2 * out_bytes + 256 * 2 ** 20
    dropped = c["B"] * c["Fo"] * Do * 56 * 56 * 4
    print(upd, precision, "peak MB", peak / 2 ** 20, "budget MB", budget / 2 ** 20, "dropped map MB", dropped / 2 ** 20)
    if precision == "tf32":                  # tf32x3 is the validation mode: its GEMMs split operands into more copies
        assert peak <= budget
    G = torch.randn(y.shape, generator=torch.Generator().manual_seed(1))
    (y * G.cuda()).sum().backward()
    torch.cuda.synchronize()
    ours = {k: t[k].grad.detach().cpu() for k in ("curr", "vf", "Wb", "Wc", "Wu") if t[k] is not None}
    yc = y.detach().cpu()
    del y, t
    torch.cuda.empty_cache()
    ref, tr = _oracle(c, p, seed, out_size, device="cuda")
    e = rel_err(yc, ref)
    print(upd, "full-size logits rel", e)
    assert e < 1e-3
    (ref * G.cuda().double()).sum().backward()
    for k, gk in ours.items():
        ek = rel_err(gk, tr[k].grad)
        print(upd, precision, "grad", k, ek)
        assert ek < (GRAD_TOL if k in ("Wb", "Wu") else 1e-3), k
