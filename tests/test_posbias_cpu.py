"""CPU checks of the --pos bias / --pos none module surface: the reference's parameter names and shapes, loading a
reference state_dict (with its index buffers) strictly, and the switches that still refuse to run."""
import ctypes as C

import pytest
import torch

import segtran_b200.networks.segtran_shared as S
from segtran_b200 import _lib, ops
from tests.helpers import encoder_config


def _cfg(pos, dims=(32, 32, 32), pos_dim=3, squeeze=False, grid=(5, 6, 7)):
    cfg = encoder_config(S.SegtranConfig, dims=list(dims), num_modes=4, num_attractors=4, pos_dim=pos_dim)
    cfg.use_squeezed_transformer = squeeze
    cfg.pos_code_type = pos
    cfg.pos_bias_radius = 2
    cfg.max_pos_size = grid
    return cfg


@pytest.mark.parametrize("pos_dim,cls", [(2, S.SlidingPosBiases2D), (3, S.SlidingPosBiases3D)])
def test_bias_parameters_follow_the_reference(pos_dim, cls):
    grid = (6, 7) if pos_dim == 2 else (5, 6, 7)
    enc = S.SegtranFusionEncoder(_cfg("bias", pos_dim=pos_dim, grid=grid), "Fusion")
    coder = enc.pos_code_layer.pos_coder
    assert isinstance(coder, cls)
    sd = enc.state_dict()
    assert sd["pos_code_layer.pos_coder.biases"].shape == (5,) * pos_dim
    assert float(sd["pos_code_layer.pos_coder.biases"].abs().sum()) == 0.0       # zero-initialised
    assert not any(k.startswith("pos_code_layer.pos_coder.all_") for k in sd)
    assert not any("pos_fc" in k for k in sd)
    assert enc.pos_code_weight == 0 and all(l.pos_code_weight == 1.0 for l in enc.translayers)


def test_pos_code_weight_reaches_the_attention_layers():
    cfg = _cfg("bias")
    cfg.pos_code_weight = 0.5
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    assert all(l.pos_code_weight == 0.5 for l in enc.translayers)


def test_seeded_construction_does_not_draw_for_the_biases():
    torch.manual_seed(0)
    a = S.SegtranFusionEncoder(_cfg("bias"), "Fusion").state_dict()
    torch.manual_seed(0)
    b = S.SegtranFusionEncoder(_cfg("none"), "Fusion").state_dict()
    for k, v in b.items():
        assert torch.equal(a[k], v), k


def test_reference_state_dict_with_index_buffers_loads_strictly():
    enc = S.SegtranFusionEncoder(_cfg("bias", grid=(3, 3, 3)), "Fusion")
    sd = dict(enc.state_dict())
    for name in ("all_h1s", "all_w1s", "all_d1s", "all_h2s", "all_w2s", "all_d2s"):
        sd["pos_code_layer.pos_coder." + name] = torch.zeros(3, 3, 3, 5, 5, 5, dtype=torch.int64)
    sd["pos_code_layer.pos_coder.biases"] = torch.randn(5, 5, 5)
    enc.load_state_dict(sd, strict=True)
    assert torch.equal(enc.pos_code_layer.pos_coder.biases.detach(), sd["pos_code_layer.pos_coder.biases"])


def test_none_has_no_positional_parameters():
    enc = S.SegtranFusionEncoder(_cfg("none", squeeze=True), "Fusion")
    assert isinstance(enc.pos_code_layer.pos_coder, S.NoneEmbedder)
    assert not any(k.startswith("pos_code_layer.") for k in enc.state_dict())
    assert enc.pos_code_layer(torch.Size((2, 2, 2)), torch.ones(1, 8, 3)) is None


def test_grid_and_radius_limits():
    with pytest.raises(ValueError):
        S.SlidingPosBiases3D(3, 0, (4, 4, 4))
    coder = S.SlidingPosBiases2D(2, 2, (6, 7))
    pb = coder(torch.Size((6, 7)))
    assert isinstance(pb, ops.PosBias) and pb.grid == (6, 7) and pb.num_tokens == 42
    with pytest.raises(ValueError):
        coder(torch.Size((6, 8)))


def test_refused_combinations():
    with pytest.raises(SystemExit):                   # the reference exits: biases need --nosqueeze
        S.SegtranFusionEncoder(_cfg("bias", squeeze=True), "Fusion")
    cfg = _cfg("bias")
    cfg.use_attn_consist_loss = True
    with pytest.raises(NotImplementedError):
        S.SegtranFusionEncoder(cfg, "Fusion")
    for pos in ("rand", "sinu"):
        with pytest.raises(NotImplementedError):
            S.SegtranFusionEncoder(_cfg(pos), "Fusion")


def test_posbias_struct_layout_matches_header():
    assert C.sizeof(_lib.sx_posbias) == 32
    assert _lib.sx_attn_probs_args.posbias.offset == 160 and C.sizeof(_lib.sx_attn_probs_args) == 192
