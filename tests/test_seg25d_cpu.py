"""Host-side checks of the 2.5-D model (segtran_b200.networks.segtran25d): configuration parity with the reference's
Segtran25dConfig, strict loading of the reference state dicts stored in the tests/golden/seg25d_*.pt fixtures (built by
oracle/gen_seg25d_golden.py from the real reference), and the documented errors."""
from __future__ import annotations

import os
from argparse import Namespace

import pytest
import torch

import segtran_b200.networks.segtran_shared as S
import segtran_b200.networks.segtran25d as M

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["seg25d_stemconv", "seg25d_updconv", "seg25d_dgroup2", "seg25d_direct34", "seg25d_posbias"]


class _Eff(torch.nn.Module):
    def extract_endpoints(self, x):
        raise AssertionError("not called")


def load_fixture(name):
    return torch.load(os.path.join(GOLDEN, name + ".pt"), map_location="cpu", weights_only=False)


def build(fx, **over):
    args = Namespace(**dict(fx["args"], **over))
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    cfg = M.Segtran25dConfig()
    cfg.update_config(args)
    cfg.max_pos_size = tuple(fx["grid"])
    return M.Segtran25d(cfg, backbone=_Eff())


def test_config_defaults_and_update_keys():
    cfg = M.Segtran25dConfig()
    assert (cfg.backbone_type, cfg.inchan_to3_scheme, cfg.D_groupsize, cfg.D_pool_K, cfg.out_fpn_upsampleD_scheme) == \
        ('eff-b3', 'stemconv', 1, 2, 'conv')
    assert cfg.in_fpn_layers == [3, 4] and cfg.out_fpn_layers == [1, 2, 3, 4] and cfg.num_attractors == 1024
    assert cfg.bb_feat_dims == S.bb2feat_dims['eff-b3'] and cfg.pos_dim == 3 and cfg.G == 8
    args = Namespace(in_fpn_layers='34', out_fpn_layers='1234', in_fpn_scheme='AN', out_fpn_scheme='AN',
                     translayer_compress_ratios=[1, 1], D_pool_K=4, D_groupsize=2, out_fpn_upsampleD_scheme='none',
                     base_initializer_range=0.05, use_attn_consist_loss=True, num_classes=4, device='cpu')
    cfg.update_config(args)
    assert (cfg.D_pool_K, cfg.D_groupsize, cfg.out_fpn_upsampleD_scheme, cfg.num_classes) == (4, 2, 'none', 4)
    assert cfg.base_initializer_range == 0.05
    assert cfg.use_attn_consist_loss is False          # not in the reference's key list: --attnconsist never reaches it


@pytest.mark.parametrize("name", CASES)
def test_reference_state_dict_loads_strictly(name):
    fx = load_fixture(name)
    net = build(fx)
    ref = fx["state_dict"]
    ours = {k: v for k, v in net.state_dict().items() if not k.startswith("backbone.")}
    ref_keys = {k for k in ref if ".pos_coder.all_" not in k}          # the reference's index buffers are not kept
    assert set(ours) == ref_keys
    for k in ours:
        assert tuple(ours[k].shape) == tuple(ref[k].shape), k
    net.load_state_dict(ref, strict=True)
    for k in ref_keys:
        assert torch.equal(net.state_dict()[k], ref[k]), k


def test_stemconv_changes_the_stem_of_its_own_backbone(monkeypatch):
    fx = load_fixture("seg25d_stemconv")
    assert fx["stem_change"] == (4, True)
    seen = {}

    class Stem(_Eff):
        def _change_in_channels(self, n, keep_RGB_weight=False):
            seen["stem"] = (n, keep_RGB_weight)

    monkeypatch.setattr(M, "_reference_backbone2d", lambda *a: Stem())
    args = Namespace(**fx["args"])
    S.bb2feat_dims[args.backbone_type] = fx["bb_feat_dims"]
    cfg = M.Segtran25dConfig()
    cfg.update_config(args)
    M.Segtran25d(cfg)
    assert seen["stem"] == (4, True)
    assert isinstance(M.Segtran25d(cfg, backbone=_Eff()).in_bridge_to3, torch.nn.Identity)


def test_unsupported_input_schemes_raise():
    fx = load_fixture("seg25d_updconv")
    with pytest.raises(NotImplementedError, match="stemconv"):
        build(fx, inchan_to3_scheme="stemconv", orig_in_channels=4)         # resnet backbone
    with pytest.raises(NotImplementedError, match="avgto3"):
        build(fx, inchan_to3_scheme="avgto3", orig_in_channels=5)
    with pytest.raises(NotImplementedError, match="not supported for scheme"):
        build(fx, inchan_to3_scheme="dup3", orig_in_channels=2)


def test_outdrop_in_training_and_ragged_sizes_raise():
    fx = load_fixture("seg25d_updconv")
    net = build(fx, out_fpn_do_dropout=True)
    feat = torch.zeros(2, 8, 16, 2, 2)
    with pytest.raises(NotImplementedError, match="outdrop"):
        net.train().hot_path(feat, None, None, (16, 16, 8))
    net = build(fx)
    with pytest.raises(ValueError, match="integer multiple"):
        net.eval().hot_path(feat, None, None, (16, 16, 9))
    with pytest.raises(ValueError, match="integer multiple"):
        net.eval().hot_path(feat, None, None, (17, 16, 8))



def oracle_inputs(fx, net):
    """The per-slice mask, the oracle's keyword arguments and the output size of a fixture."""
    from oracle import seg25d_oracle as SO
    a = fx["args"]
    p = fx["state_dict"]
    x = fx["batch"]
    B, C, H, W, D = x.shape
    g = a["D_groupsize"]
    if g > 1:
        x = x.view(B, C, H, W, -1, g).permute(0, 1, 5, 2, 3, 4).reshape(B, C * g, H, W, -1)
    if "in_bridge_to3.weight" in p:
        x = torch.nn.functional.conv3d(x, p["in_bridge_to3.weight"], p["in_bridge_to3.bias"])
    kw = dict(in_layers=net.in_fpn_layers, out_layers=net.out_fpn_layers, translayer_dims=net.translayer_dims,
              num_modes=a["num_modes"], D_pool_K=a["D_pool_K"], upd=a["out_fpn_upsampleD_scheme"])
    return SO.get_mask(x, 8), kw, (H, W, D)


@pytest.mark.parametrize("name", ["seg25d_stemconv", "seg25d_updconv", "seg25d_dgroup2", "seg25d_direct34"])
def test_oracle_matches_reference_fixture(name):
    from oracle import seg25d_oracle as SO
    fx = load_fixture(name)
    net = build(fx)
    mask, kw, out_size = oracle_inputs(fx, net)
    if name == "seg25d_stemconv":
        assert int(mask.sum()) < mask.numel()                          # the zero slab masks tokens
    y = SO.forward(fx["state_dict"], fx["feats"], mask, fx["batch"].shape[0], out_size, **kw)
    assert y.shape == fx["out"].shape
    assert float((y - fx["out"]).abs().max() / fx["out"].abs().max()) < 1e-5


def test_oracle_unfolds_depth_as_slice_times_dk_plus_j():
    """--upd conv: channel f*Dk + j of out_fpn_upsampleD at slice i lands at depth i*Dk + j (segtran25d.py:357-362)."""
    from oracle import seg25d_oracle as SO
    Fo, Dk, D2 = 2, 3, 4
    x = torch.zeros(1, Fo * Dk, 1, 1, D2)
    x[0, 0, 0, 0, :] = torch.arange(D2, dtype=torch.float32)           # channel 0 carries the slice index i
    w = torch.zeros(Fo * Dk, Fo * Dk, 1, 1, 1)
    w[:, 0] = 1.0
    b = torch.tensor([100. * (c // Dk) + 10. * (c % Dk) for c in range(Fo * Dk)])
    y = SO.depth_map({"out_fpn_upsampleD.weight": w, "out_fpn_upsampleD.bias": b}, x, Dk, "conv")
    assert y.shape == (1, Fo, 1, 1, D2 * Dk)
    for f in range(Fo):
        for i in range(D2):
            for j in range(Dk):
                assert float(y[0, f, 0, 0, i * Dk + j]) == 100. * f + 10. * j + i
