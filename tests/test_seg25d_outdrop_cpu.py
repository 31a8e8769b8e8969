"""Host-side checks of the 2.5-D --outdrop head (ops.seg_head_slices_dropout, csrc/sx_head_drop.cu with a slice-major
source): the float64 oracle (oracle/seg25d_outdrop_oracle.py) against the tests/golden/seg25d_outdrop_*.pt fixtures built
from the real reference by oracle/gen_seg25d_outdrop_golden.py, the layout and depth-map declarations of the header
and the ctypes binding, and the argument errors raised before any launch."""
from __future__ import annotations

import ctypes
import os
import re
from argparse import Namespace

import pytest
import torch

import segtran_b200.networks.segtran_shared as S
import segtran_b200.networks.segtran25d as M
from oracle import head_oracle as HO
from oracle import seg25d_outdrop_oracle as DO
from oracle import seg25d_oracle as SO
from segtran_b200 import _lib as L
from tests.helpers import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["seg25d_outdrop_updconv", "seg25d_outdrop_interp", "seg25d_outdrop_noupd", "seg25d_outdrop_dk1",
         "seg25d_outdrop_k5"]


class _Eff(torch.nn.Module):
    def extract_endpoints(self, x):
        raise AssertionError("not called")


def build(fx, **over):
    args = Namespace(**dict(fx["args"], **over))
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    cfg = M.Segtran25dConfig()
    cfg.update_config(args)
    cfg.max_pos_size = tuple(fx["grid"])
    return M.Segtran25d(cfg, backbone=_Eff())


def oracle_inputs(fx, net):
    a = fx["args"]
    p = fx["state_dict"]
    x = fx["batch"]
    B, C, H, W, D = x.shape
    if "in_bridge_to3.weight" in p:
        x = torch.nn.functional.conv3d(x, p["in_bridge_to3.weight"], p["in_bridge_to3.bias"])
    kw = dict(in_layers=net.in_fpn_layers, out_layers=net.out_fpn_layers, translayer_dims=net.translayer_dims,
              num_modes=a["num_modes"], D_pool_K=a["D_pool_K"], upd=a["out_fpn_upsampleD_scheme"])
    return SO.get_mask(x, 8), kw, (H, W, D)


def test_fixture_set_covers_the_cases():
    seen = set()
    for name in NAMES:
        fx = load_golden(name)
        a = fx["args"]
        assert fx["train"] and a["out_fpn_do_dropout"] and a["dropout_prob"] == 0.0, name
        seen.add((a["out_fpn_upsampleD_scheme"], a["D_pool_K"], a["num_classes"]))
    assert ("conv", 2, 3) in seen and ("interpolate", 2, 2) in seen and ("interp", 2, 2) in seen
    assert ("conv", 1, 2) in seen and ("conv", 2, 5) in seen


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fixture(name):
    fx = load_golden(name)
    net = build(fx)
    mask, kw, out_size = oracle_inputs(fx, net)
    y = DO.forward(fx["state_dict"], fx["feats"], mask, fx["batch"].shape[0], out_size, **kw)
    assert y.shape == fx["out"].shape
    assert float((y - fx["out"]).abs().max() / fx["out"].abs().max()) < 1e-5


@pytest.mark.parametrize("name", NAMES)
def test_reference_state_dict_loads_strictly(name):
    fx = load_golden(name)
    net = build(fx)
    net.load_state_dict(fx["state_dict"], strict=True)
    assert net.out_fpn_do_dropout and net.out_fpn_dropout.p == 0.0


def test_oracle_keep_mask_layout():
    """keep is [B,F',D',H1,W1]: dropping channel f at output depth d' zeroes exactly that (f, d') plane of the map the
    class conv reads, here checked through a class conv that picks channel f."""
    g = torch.Generator().manual_seed(3)
    B, D2, Cf, F_, H1, W1, Dk = 1, 3, 4, 6, 2, 2, 2
    curr = torch.randn(B * D2, Cf, H1, W1, generator=g)
    vf = torch.randn(B, 1 * 1 * 3, F_, generator=g)
    Wb, bb = torch.randn(F_, Cf, generator=g), torch.randn(F_, generator=g)
    Wu, bu = torch.randn(F_, F_, generator=g), torch.randn(F_, generator=g)
    Fo = F_ // Dk
    Wc = torch.zeros(1, Fo)
    Wc[0, 1] = 1.0
    full = DO.head_25d(curr, vf, (1, 1, 3), Wb, bb, Wc, None, (H1, W1, D2 * Dk), Dk, "conv", Wu, bu)
    keep = torch.ones(B, Fo, D2 * Dk, H1, W1, dtype=torch.float64)
    keep[0, 1, 4] = 0.0
    dropped = DO.head_25d(curr, vf, (1, 1, 3), Wb, bb, Wc, None, (H1, W1, D2 * Dk), Dk, "conv", Wu, bu,
                          keep=keep, p=0.5)
    assert torch.allclose(dropped[..., 4], torch.zeros_like(dropped[..., 4]))
    others = [d for d in range(D2 * Dk) if d != 4]
    assert torch.allclose(dropped[..., others], 2.0 * full[..., others])


def test_header_and_ctypes_declare_the_layout_and_the_interleaved_unfold():
    hdr = open(os.path.join(ROOT, "include", "segtran_b200.h")).read()
    assert re.search(r"SX_HEAD_DMAP_UNFOLD_INTERLEAVED = 3", hdr)
    assert re.search(r"SX_HEAD_SRC_DEPTH_MAJOR = 0, SX_HEAD_SRC_SLICE_MAJOR = 1", hdr)
    assert re.search(r"int32_t src_layout;", hdr) and "_pad;" not in hdr[hdr.index("SX_HEAD_SRC_DEPTH_MAJOR = 0"):
                                                                          hdr.index("} sx_head_dropout_args;")]
    assert (L.SX_HEAD_DMAP_NONE, L.SX_HEAD_DMAP_INTERP, L.SX_HEAD_DMAP_UNFOLD, L.SX_HEAD_DMAP_UNFOLD_INTERLEAVED) == \
        (0, 1, 2, 3)
    assert (L.SX_HEAD_SRC_DEPTH_MAJOR, L.SX_HEAD_SRC_SLICE_MAJOR) == (0, 1)
    assert L.sx_head_dropout_args.src_layout.offset == 44 and L.sx_head_dropout_args.K.offset == 40
    assert L.sx_head_dropout_args.part_floats.offset == 96 and ctypes.sizeof(L.sx_head_dropout_args) == 104
    assert L.sx_head_dropout_args().src_layout == L.SX_HEAD_SRC_DEPTH_MAJOR          # zero-initialised callers


def _case(B=1, D2=4, Cf=8, Fd=8, H1=4, W1=4, grid=(2, 2, 2), K=2):
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.randn(*s, generator=g)                     # noqa: E731
    N = grid[0] * grid[1] * grid[2]
    return dict(curr=r(B * D2, Cf, H1, W1), vf=r(B, N, Fd), Wb=r(Fd, Cf, 1, 1, 1), bb=r(Fd), Wc=r(K, Fd // 2, 1, 1, 1),
                bc=r(K), Wu=r(Fd, Fd, 1, 1, 1), bu=r(Fd), grid=grid)


def test_argument_errors_before_any_launch():
    from segtran_b200 import ops
    c = _case()
    args = lambda **o: dict(dict(c, out_size=(8, 8, 8), p=0.2, d_pool_k=2, upsample_d="conv"), **o)   # noqa: E731

    def call(**o):
        a = args(**o)
        return ops.seg_head_slices_dropout(a["curr"], a["vf"], a["grid"], a["Wb"], a["bb"], a["Wc"], a["bc"],
                                           a["out_size"], a["p"], a["d_pool_k"], a["upsample_d"], Wu=a["Wu"],
                                           bu=a["bu"])
    with pytest.raises(ValueError, match="multiple of the batch"):
        call(vf=torch.zeros(3, 8, 8))
    with pytest.raises(ValueError, match="does not hold"):
        call(grid=(2, 2, 3))
    with pytest.raises(ValueError, match="dropout probability"):
        call(p=1.0)
    with pytest.raises(ValueError, match="needs out_fpn_upsampleD"):
        call(Wu=None)
    with pytest.raises(ValueError, match="D_pool_K"):
        call(Wu=torch.zeros(6, 8, 1, 1, 1))
    with pytest.raises(ValueError, match="class conv reads"):
        call(upsample_d="interpolate")                               # Wc has F/2 columns: only 'conv' halves F
    with pytest.raises(ValueError, match=r"\(H, W, D\)"):
        call(out_size=(8, 8))
    with pytest.raises(ValueError, match="curr"):
        call(curr=torch.zeros(4, 8, 16))
    with pytest.raises(L.SxError):                                   # valid arguments on the CPU: no fallback
        call()


def test_kernel_argument_errors():
    """sx_head_dropout_fwd/bwd refuse an unknown layout or depth map and an interleaved unfold whose channels do not
    split into D_pool_K groups before reading any pointer."""
    a = L.sx_head_dropout_args()
    a.src, a.Wc, a.B, a.Fs, a.Ds, a.Fo, a.HW, a.Dk, a.K, a.p = 16, 16, 1, 8, 2, 4, 16, 2, 1, 0.1
    a.dmap, a.src_layout = L.SX_HEAD_DMAP_UNFOLD_INTERLEAVED, 2
    with pytest.raises(L.SxError, match="source layout"):
        L.call("sx_head_dropout_fwd", ctypes.byref(a), 16, None)
    a.src_layout, a.dmap = L.SX_HEAD_SRC_SLICE_MAJOR, 4
    with pytest.raises(L.SxError, match="depth map"):
        L.call("sx_head_dropout_fwd", ctypes.byref(a), 16, None)
    a.dmap, a.Fs = L.SX_HEAD_DMAP_UNFOLD_INTERLEAVED, 7
    with pytest.raises(L.SxError, match="unfold"):
        L.call("sx_head_dropout_bwd", ctypes.byref(a), 16, 16, 0, 16, None)


def test_outdrop_in_training_wants_cuda_tensors_after_the_size_check():
    """--outdrop in training runs on the CUDA dropout head; host tensors are refused before any work, and a token grid
    the input size is not a multiple of raises ValueError first, in training as in evaluation."""
    fx = load_golden("seg25d_outdrop_updconv")
    net = build(fx)
    assert net.out_fpn_do_dropout
    feat = torch.zeros(2, 8, 16, 2, 2)
    with pytest.raises(NotImplementedError, match="CUDA dropout head"):
        net.train().hot_path(feat, None, None, (16, 16, 8))
    for mode in (net.train, net.eval):
        mode()
        with pytest.raises(ValueError, match="integer multiple"):
            net.hot_path(feat, None, None, (16, 16, 9))
        with pytest.raises(ValueError, match="integer multiple"):
            net.hot_path(feat, None, None, (17, 16, 8))


def test_outdrop_with_the_direct_head_is_accepted():
    """--outfpn equal to --infpn: the reference builds no out-FPN dropout and --outdrop does nothing."""
    fx = load_golden("seg25d_direct34")
    net = build(fx, out_fpn_do_dropout=True)
    assert not net.do_out_fpn and not hasattr(net, "out_fpn_dropout")
    net.load_state_dict(fx["state_dict"], strict=True)


def test_keep_mask_regeneration_matches_the_hash():
    """The oracle's keep_mask is drop_keep1 over the flat [B,F',D',H1,W1] index (the same mask for either layout)."""
    m = HO.keep_mask(5, (1, 2, 3, 2, 2), 0.3)
    flat = HO.drop_keep1(5, torch.arange(24).numpy(), 0.3)
    assert torch.equal(m.reshape(-1).bool(), torch.from_numpy(flat))


def test_torch_keep_mask_matches_the_numpy_hash():
    for seed, p in ((5, 0.3), (2 ** 63 + 12345, 0.1), (987654321, 0.5)):
        shape = (2, 3, 4, 5, 7)
        assert torch.equal(DO.keep_mask_torch(seed, shape, p, "cpu"), HO.keep_mask(seed, shape, p).bool())
