"""CPU checks of the class head without the out-FPN (out_fpn_layers == in_fpn_layers): the module surface against the
reference fixtures (oracle/gen_direct_head_golden.py) — state_dict keys and shapes, seeded-construction digests, strict
checkpoint loading — the '234' quirk, the no-op options, and the float64 oracle against each fixture's logits."""
from argparse import Namespace

import pytest
import torch
import torch.nn.functional as F

from oracle import direct_head_oracle as DO
from oracle import segtran_oracle as O
from tests.helpers import load_golden, rel_err

TOL = 1e-4
NAMES2 = ["seg2d_direct34", "seg2d_direct234"]
NAMES3 = ["seg3d_direct34", "seg3d_direct34_outdrop"]


class _BackboneRngStandIn(torch.nn.Module):
    """Leaves the torch RNG where the reference's I3D backbone leaves it after construction and init_weights."""

    def __init__(self, fx):
        super().__init__()
        self.fx, self.applied = fx, False
        torch.set_rng_state(fx["rng_built"])

    def apply(self, fn):
        if not self.applied:
            torch.set_rng_state(self.fx["rng_applied"])
            self.applied = True
        return self


def _shell(fx, monkeypatch, seeded=True, **overrides):
    import segtran_b200.networks.segtran_shared as S
    args = Namespace(**dict(fx["args"], **overrides))
    if fx["kind"] == "seg3d":
        import segtran_b200.networks.segtran3d as M
        monkeypatch.setitem(S.bb2feat_dims, "i3d-tiny", fx["bb_feat_dims"])
        monkeypatch.setattr(M, "_reference_i3d", lambda do_pool1, use_pretrained: _BackboneRngStandIn(fx))
        if seeded:
            torch.manual_seed(fx["init_seed"])
        cfg = M.Segtran3dConfig()
        cfg.update_config(args)
        return M.Segtran3d(cfg)
    import segtran_b200.networks.segtran2d as M
    monkeypatch.setitem(S.bb2feat_dims, "resnet-tiny", fx["bb_feat_dims"])
    if seeded:
        torch.manual_seed(fx["init_seed"])
    cfg = M.Segtran2dConfig()
    cfg.update_config(args)
    return M.Segtran2d(cfg, backbone=torch.nn.Identity())          # the reference's stand-in draws no numbers


@pytest.mark.parametrize("name", NAMES2 + NAMES3)
def test_module_surface_digests_and_strict_load(name, monkeypatch):
    from oracle.gen_golden import _digest
    fx = load_golden(name)
    net = _shell(fx, monkeypatch)
    assert not net.do_out_fpn
    sd = {k: v for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in fx["state_dict"].items()}
    diff = [k for k in sd if _digest(sd[k]) != fx["init_digests"][k]]
    assert not diff, diff[:5]
    assert not any(k.startswith(("out_fpn", "out_gn", "out_bn")) for k in sd)
    net.load_state_dict(fx["state_dict"], strict=True)


def test_234_builds_the_transposed_conv(monkeypatch):
    fx = load_golden("seg2d_direct234")
    net = _shell(fx, monkeypatch)
    assert net.in_fpn_layers == [2, 3, 4] and isinstance(net.out_conv, torch.nn.ConvTranspose2d)
    C, K = fx["bb_feat_dims"][4], fx["args"]["num_classes"]
    assert tuple(net.out_conv.weight.shape) == (C, K, 2, 2)


def test_outdrop_and_upd_conv_are_accepted(monkeypatch):
    fx3 = load_golden("seg3d_direct34")
    net = _shell(fx3, monkeypatch, seeded=False, out_fpn_upsampleD_scheme="conv", out_fpn_do_dropout=True)
    assert isinstance(net.out_conv3d, torch.nn.ConvTranspose3d)
    assert tuple(net.out_conv3d.weight.shape)[2:] == (2, 2, 1)
    assert not hasattr(net, "out_fpn_upsampleD") and not hasattr(net, "out_fpn_dropout")
    net.load_state_dict(fx3["state_dict"], strict=True)
    net2 = _shell(load_golden("seg2d_direct34"), monkeypatch, seeded=False, out_fpn_do_dropout=True)
    assert isinstance(net2.out_conv, torch.nn.ConvTranspose2d) and not hasattr(net2, "out_fpn_dropout")


def _stage(conv, cur, hi, norm_w, norm_b, mode):
    y = conv(cur) + F.interpolate(hi, size=cur.shape[2:], mode=mode, align_corners=False)
    return F.group_norm(y, 8, norm_w, norm_b)


@pytest.mark.parametrize("name", NAMES2)
def test_oracle_matches_seg2d_fixture(name):
    fx = load_golden(name)
    p, f, a = fx["state_dict"], fx["feats"], fx["args"]
    layers = [int(c) for c in a["in_fpn_layers"]]
    cur = f[layers[0]]
    for lv in layers[:-1]:
        conv = lambda x, lv=lv: F.conv2d(x, p["in_fpn%d%d_conv.weight" % (lv, lv + 1)],       # noqa: E731
                                         p["in_fpn%d%d_conv.bias" % (lv, lv + 1)])
        cur = _stage(conv, cur, f[lv + 1], p["in_gn%db.weight" % (lv + 1)], p["in_gn%db.bias" % (lv + 1)], "bilinear")
    grid = tuple(cur.shape[2:])
    B, S = cur.shape[0], fx["batch"].shape[-1]
    vmask = (F.avg_pool2d(fx["batch"].abs(), 2 ** layers[0]).sum(1) > 0).reshape(B, -1, 1)
    pos = O.voxels_pos_for_grid(grid, (S // grid[0], S // grid[1]), B)
    Fd = fx["bb_feat_dims"][4]
    fused = O.fusion_encoder(p, "voxel_fusion.", O.flatten_tokens(cur), pos, vmask, [Fd, Fd], a["num_modes"])
    y = DO.direct_head(O.scatter_tokens(fused, grid), p["out_conv.weight"], p["out_conv.bias"], (S, S))
    assert y.shape == fx["out"].shape
    assert rel_err(y, fx["out"]) < TOL


@pytest.mark.parametrize("name", NAMES3)
def test_oracle_matches_seg3d_fixture(name):
    fx = load_golden(name)
    p, f, a = fx["state_dict"], fx["feats"], fx["args"]
    conv = lambda x: F.conv3d(x, p["in_fpn34_conv.weight"], p["in_fpn34_conv.bias"])       # noqa: E731
    cur = _stage(conv, f[3], f[4], p["in_gn4b.weight"], p["in_gn4b.bias"], "trilinear")
    sz = list(cur.shape[2:])
    sz[0] //= a["D_pool_K"]
    feat_fpn = F.interpolate(cur, size=sz, mode="trilinear", align_corners=False)
    grid = tuple(feat_fpn.shape[2:])
    B = feat_fpn.shape[0]
    H, W, D = fx["batch"].shape[2:]
    assert grid[0] != grid[1]
    pos = O.voxels_pos_for_grid(grid, (D // grid[0], H // grid[1], W // grid[2]), B)
    vmask = torch.ones(B, feat_fpn[0, 0].numel(), 1, dtype=torch.long)
    Fd = fx["bb_feat_dims"][4]
    fused = O.fusion_encoder(p, "voxel_fusion.", O.flatten_tokens(feat_fpn), pos, vmask, [Fd, Fd], a["num_modes"])
    y = DO.direct_head(O.scatter_tokens(fused, grid), p["out_conv3d.weight"], p["out_conv3d.bias"], (H, W, D))
    assert y.shape == fx["out"].shape
    assert rel_err(y, fx["out"]) < TOL


def test_abi_has_subpixel_entries():
    from segtran_b200 import _lib as L
    assert "sx_subpixel_resize_fwd" in L.EXPORTS and "sx_subpixel_resize_bwd" in L.EXPORTS
    assert len(L._PROTOS["sx_subpixel_resize_fwd"]) == 12 and len(L._PROTOS["sx_subpixel_resize_bwd"]) == 11
