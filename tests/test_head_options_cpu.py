"""CPU checks of the head options --upd conv and --outdrop: the float64 head oracle against the fixtures the real
reference shells produced (oracle/gen_head_golden.py), seeded construction and strict checkpoint loading of
out_fpn_upsampleD, and the C ABI entries of the dropout head."""
import ctypes
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import head_oracle as HO
from oracle import segtran_oracle as O
from tests.helpers import load_golden, rel_err

TOL = 1e-4
NAMES3 = ["seg3d_updconv", "seg3d_outdrop", "seg3d_updconv_outdrop"]


def _fpn3d(fx):
    p, f = fx["state_dict"], fx["feats"]
    cur = F.conv3d(f[3], p["in_fpn34_conv.weight"], p["in_fpn34_conv.bias"])
    cur = cur + F.interpolate(f[4], size=cur.shape[2:], mode="trilinear", align_corners=False)
    cur = F.group_norm(cur, 8, p["in_gn4b.weight"], p["in_gn4b.bias"])
    sz = list(cur.shape[2:]); sz[0] //= 2
    feat_fpn = F.interpolate(cur, size=sz, mode="trilinear", align_corners=False)
    c = F.conv3d(f[1], p["out_fpn12_conv3d.weight"], p["out_fpn12_conv3d.bias"])
    c = F.group_norm(c + F.interpolate(f[2], size=c.shape[2:], mode="trilinear", align_corners=False), 8,
                     p["out_gn2b.weight"], p["out_gn2b.bias"])
    c2 = F.conv3d(c, p["out_fpn23_conv3d.weight"], p["out_fpn23_conv3d.bias"])
    c2 = F.group_norm(c2 + F.interpolate(f[3], size=c2.shape[2:], mode="trilinear", align_corners=False), 8,
                      p["out_gn3b.weight"], p["out_gn3b.bias"])
    return feat_fpn, c2


@pytest.mark.parametrize("name", NAMES3)
def test_head_oracle_matches_seg3d_fixture(name):
    fx = load_golden(name)
    a = fx["args"]
    p = fx["state_dict"]
    feat_fpn, curr = _fpn3d(fx)
    B, grid = feat_fpn.shape[0], tuple(feat_fpn.shape[2:])
    Fd, M = fx["bb_feat_dims"][4], a["num_modes"]
    S = fx["batch"].shape[-1]
    pos = O.voxels_pos_for_grid(grid, (S // grid[0], S // grid[1], S // grid[2]), B)
    vmask = torch.ones(B, feat_fpn[0, 0].numel(), 1, dtype=torch.long)
    fused = O.fusion_encoder(p, "voxel_fusion.", O.flatten_tokens(feat_fpn), pos, vmask, [Fd, Fd], M)
    vmap = O.scatter_tokens(fused, grid)
    up = a["out_fpn_upsampleD_scheme"]
    Dk = a["D_pool_K"]
    Fo = Fd // Dk if up == "conv" else Fd
    keep = torch.ones(B, Fo, curr.shape[2] * Dk, *curr.shape[3:]) if fx["train"] else None
    y = HO.seg_head_3d(curr, vmap, p["out_fpn_bridgeconv3d.weight"], p["out_fpn_bridgeconv3d.bias"],
                       p["out_conv3d.weight"], p["out_conv3d.bias"], (S, S, S), Dk, up,
                       p.get("out_fpn_upsampleD.weight"), p.get("out_fpn_upsampleD.bias"), keep=keep, p=0.0)
    assert rel_err(y, fx["out"]) < TOL


def test_head_oracle_matches_seg2d_fixture():
    fx = load_golden("seg2d_outdrop")
    p, f = fx["state_dict"], fx["feats"]
    cur = F.conv2d(f[3], p["in_fpn34_conv.weight"], p["in_fpn34_conv.bias"])
    cur = cur + F.interpolate(f[4], size=cur.shape[2:], mode="bilinear", align_corners=False)
    feat_fpn = F.group_norm(cur, 8, p["in_gn4b.weight"], p["in_gn4b.bias"])
    c = F.conv2d(f[1], p["out_fpn12_conv.weight"], p["out_fpn12_conv.bias"])
    c = F.group_norm(c + F.interpolate(f[2], size=c.shape[2:], mode="bilinear", align_corners=False), 8,
                     p["out_gn2b.weight"], p["out_gn2b.bias"])
    c2 = F.conv2d(c, p["out_fpn23_conv.weight"], p["out_fpn23_conv.bias"])
    c2 = F.group_norm(c2 + F.interpolate(f[3], size=c2.shape[2:], mode="bilinear", align_corners=False), 8,
                      p["out_gn3b.weight"], p["out_gn3b.bias"])
    vmask = (F.avg_pool2d(fx["batch"].abs(), 8).sum(1) > 0).reshape(2, -1, 1)
    grid = tuple(feat_fpn.shape[2:])
    S = fx["batch"].shape[-1]
    pos = O.voxels_pos_for_grid(grid, (S // grid[0], S // grid[1]), 2)
    Fd = fx["bb_feat_dims"][4]
    fused = O.fusion_encoder(p, "voxel_fusion.", O.flatten_tokens(feat_fpn), pos, vmask, [Fd, Fd],
                             fx["args"]["num_modes"])
    keep = torch.ones(2, Fd, *c2.shape[2:])
    y = HO.seg_head_2d(c2, O.scatter_tokens(fused, grid), p["out_fpn_bridgeconv.weight"], p["out_fpn_bridgeconv.bias"],
                       p["out_conv.weight"], p["out_conv.bias"], (S, S), keep=keep, p=0.0)
    assert rel_err(y, fx["out"]) < TOL


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


@pytest.mark.parametrize("name", ["seg3d_updconv", "seg3d_updconv_outdrop"])
def test_updconv_seeded_construction_and_strict_load(name, monkeypatch):
    from oracle.gen_golden import _digest
    import segtran_b200.networks.segtran_shared as S
    import segtran_b200.networks.segtran3d as M3
    fx = load_golden(name)
    monkeypatch.setitem(S.bb2feat_dims, "i3d-tiny", fx["bb_feat_dims"])
    monkeypatch.setattr(M3, "_reference_i3d", lambda do_pool1, use_pretrained: _BackboneRngStandIn(fx))
    torch.manual_seed(fx["init_seed"])
    cfg = M3.Segtran3dConfig()
    cfg.update_config(Namespace(**fx["args"]))
    net = M3.Segtran3d(cfg)
    sd = {k: v for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    assert sorted(sd) == sorted(fx["init_digests"])
    diff = [k for k in sd if _digest(sd[k]) != fx["init_digests"][k]]
    assert not diff, diff[:5]
    Fd, K = fx["bb_feat_dims"][4], fx["args"]["num_classes"]
    assert tuple(net.out_fpn_upsampleD.weight.shape) == (Fd, Fd, 1, 1, 1)
    assert tuple(net.out_conv3d.weight.shape)[:2] == (K, Fd // 2)
    # a reference checkpoint loads strictly into a shell with a stand-in backbone
    net2 = M3.Segtran3d(cfg, backbone=torch.nn.Identity())
    net2.load_state_dict(fx["state_dict"], strict=True)


def test_abi_has_dropout_head_entries():
    from segtran_b200 import _lib as L
    assert "sx_head_dropout_fwd" in L.EXPORTS and "sx_head_dropout_bwd" in L.EXPORTS
    hdr = open(L.__file__.replace("segtran_b200/_lib.py", "include/segtran_b200.h")).read()
    assert "sx_head_dropout_args" in hdr and "int sx_head_dropout_fwd(" in hdr and "int sx_head_dropout_bwd(" in hdr
    assert L.sx_head_dropout_args.part_floats.offset == 96 and ctypes.sizeof(L.sx_head_dropout_args) == 104


def test_drop_keep1_restatement_keep_rate():
    """The NumPy restatement of the mask hash keeps ~1-p of the elements, independently across neighbours."""
    k = HO.drop_keep1(12345, np.arange(1 << 18, dtype=np.uint64), 0.3)
    assert abs(k.mean() - 0.7) < 0.005
    assert abs((k[1:] & k[:-1]).mean() - 0.49) < 0.006
    assert HO.drop_keep1(7, np.arange(1000, dtype=np.uint64), 0.0).all()
