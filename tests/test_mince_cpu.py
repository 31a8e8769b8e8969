"""CPU checks of the mince transformer's module surface: the reference's parameter names and shapes, the switches that
refuse to run, bad scales, and the new C ABI entry points."""
import os

import pytest
import torch

import segtran_b200.networks.segtran_shared as S
from segtran_b200 import _lib, ops
from tests.helpers import encoder_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(pos="bias", dims=(32, 32), pos_dim=3, grid=(5, 6, 7), scales=(1, 2), props=(3, 1), squeeze=False):
    cfg = encoder_config(S.SegtranConfig, dims=list(dims), num_modes=4, num_attractors=4, pos_dim=pos_dim)
    cfg.use_squeezed_transformer = squeeze
    cfg.use_mince_transformer = True
    cfg.mince_scales = None if scales is None else list(scales)
    cfg.mince_channel_props = None if props is None else list(props)
    cfg.pos_code_type = pos
    cfg.pos_bias_radius = 2
    cfg.max_pos_size = grid
    return cfg


def test_parameters_follow_the_reference():
    enc = S.SegtranFusionEncoder(_cfg(), "Fusion")
    sd = enc.state_dict()
    assert not hasattr(enc, "pos_code_layer")
    for s in range(2):
        assert sd["pos_code_layers.%d.pos_coder.biases" % s].shape == (5, 5, 5)
    layer = enc.translayers[0]
    assert isinstance(layer, S.CrossMinceAttFeatTrans) and not isinstance(layer, S.CrossAttFeatTrans)
    assert [n for n, _ in layer.named_children()] == ["query", "key", "out_trans", "att_dropout"]
    assert sd["translayers.0.key.weight"].shape == sd["translayers.0.query.weight"].shape == (32, 32)
    assert layer.mince_qk_channel_indices == [0, 4, 8]
    assert layer.out_trans.mince_channel_indices == [0, 24, 32]
    enc.apply(S.SegtranInitWeights(_cfg()).tie_qk)
    assert layer.key.weight is not layer.query.weight            # untied: not a CrossAttFeatTrans


def test_lsinu_keeps_one_positional_code_and_none_has_none():
    enc = S.SegtranFusionEncoder(_cfg("lsinu"), "Fusion")
    assert "pos_code_layer.pos_coder.pos_fc.weight" in enc.state_dict() and not hasattr(enc, "pos_code_layers")
    enc = S.SegtranFusionEncoder(_cfg("none"), "Fusion")
    assert len(enc.pos_code_layers) == 2 and not any(k.startswith("pos_code_layers") for k in enc.state_dict())


def test_channel_windows():
    assert S.fracs_to_indices(256, [1, 1, 1]) == ([0, 85, 170, 256], [85, 85, 86])
    assert S.fracs_to_indices(32, [1, 1, 2]) == ([0, 8, 16, 32], [8, 8, 16])
    assert S.mince_grids((5, 6, 7), [1, 2]) == [(5, 6, 7), (2, 3, 3)]
    assert S.mince_grids((9, 10), [1, 3]) == [(9, 10), (3, 3)]
    assert ops.down_ratio(2) == 2.0 and ops.down_ratio(3) == 3.0


def test_refused_combinations():
    with pytest.raises(SystemExit):                       # the reference exits: mince needs --nosqueeze
        S.SegtranFusionEncoder(_cfg(squeeze=True), "Fusion")
    cfg = _cfg()
    cfg.use_attn_consist_loss = True
    with pytest.raises(NotImplementedError):
        S.SegtranFusionEncoder(cfg, "Fusion")
    with pytest.raises(NotImplementedError):
        S.SqueezedAttFeatTrans(_cfg("lsinu"), "sq")
    for pos in ("rand", "sinu"):
        with pytest.raises(NotImplementedError):
            S.SegtranFusionEncoder(_cfg(pos), "Fusion")


def test_bad_scales_raise_value_error():
    with pytest.raises(ValueError):
        S.SegtranFusionEncoder(_cfg(scales=None), "Fusion")
    with pytest.raises(ValueError):
        S.SegtranFusionEncoder(_cfg(props=None), "Fusion")
    with pytest.raises(ValueError):                        # an axis of 5 cells at scale 6 is empty
        S.mince_grids((5, 6, 7), [1, 6])
    with pytest.raises(ValueError):                        # int(33 / 1.1) = 29 but floor(33 * (1 / 1.1)) = 30
        S.mince_grids((33, 4), [1, 1.1])
    enc = S.SegtranFusionEncoder(_cfg("lsinu", scales=(1, 8), props=(1, 1)), "Fusion")
    with pytest.raises(ValueError):                        # checked before anything runs on a device
        enc.translayers[0](torch.zeros(1, 210, 32), (5, 6, 7))


def test_new_entry_points_are_declared():
    with open(os.path.join(ROOT, "include", "segtran_b200.h")) as f:
        hdr = f.read()
    for name in ("sx_resize_tokens_fwd", "sx_resize_tokens_bwd"):
        assert name + "(" in hdr
        assert name in _lib.EXPORTS and name in _lib._PROTOS
    assert "sx_resample_grid" in hdr
