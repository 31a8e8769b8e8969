"""CPU checks of the mince transformer against fixtures made by the reference (oracle/gen_mince_golden.py): the float64
oracle reproduces the reference's outputs, gradients and per-scale max_attn, and seeded construction gives the
reference's initial parameters bit for bit."""
import hashlib
import os

import pytest
import torch

import segtran_b200.networks.segtran_shared as S
from oracle import mince_oracle as MO
from tests.helpers import encoder_config

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["mince3d", "mince2d", "mince_lsinu", "mince_none", "mince_clamp"]


def _load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def mince_cfg(fx):
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"], num_attractors=fx["num_attractors"],
                         pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"])
    cfg.use_squeezed_transformer = False
    cfg.use_mince_transformer = True
    cfg.mince_scales = list(fx["mince_scales"])
    cfg.mince_channel_props = list(fx["mince_channel_props"])
    cfg.pos_code_type = fx["pos_code_type"]
    cfg.pos_bias_radius = fx["pos_bias_radius"]
    cfg.pos_code_weight = fx["pos_code_weight"]
    cfg.max_pos_size = tuple(fx["grid"])
    return cfg


def _digest(t):
    t = t.detach().cpu().contiguous()
    return tuple(t.shape), str(t.dtype), hashlib.sha256(t.numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fixture(name):
    fx = _load(name)
    p = {k: v.double().requires_grad_() for k, v in fx["state_dict"].items() if v.is_floating_point()}
    x = fx["x"].double().requires_grad_()
    stats = {}
    y = MO.fusion_encoder_mince(p, "", x, fx["voxels_pos"].double(), fx["vmask"], fx["dims"], fx["num_modes"],
                                fx["pos_code_type"], fx["grid"], fx["mince_scales"], fx["mince_channel_props"],
                                pos_bias_radius=fx["pos_bias_radius"], pos_code_weight=fx["pos_code_weight"], collect=stats)
    ref = fx["out"].double()
    assert float((y.detach() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    (y * fx["G"].double()).sum().backward()
    gx = fx["grad_x"].double()
    assert float((x.grad - gx).abs().max()) <= 1e-4 * float(gx.abs().max())
    for k, g in fx["grad_params"].items():
        g = g.double()
        assert p[k].grad is not None, k
        assert float((p[k].grad - g).abs().max()) <= 1e-4 * float(g.abs().max()) + 1e-5, k
    for ours, theirs in zip(stats["max_attn"], fx["max_attn"]):
        assert ours == pytest.approx(theirs, rel=1e-4, abs=1e-6)
    if fx["pos_code_type"] == "bias":
        for s in range(len(fx["mince_scales"])):
            assert "pos_code_layers.%d.pos_coder.biases" % s in fx["grad_params"]


def test_clamp_fixture_clamps_one_scale_only():
    fx = _load("mince_clamp")
    assert fx["clamp_count"] == [[1, 0]]
    assert fx["max_attn"][0][0] > 500 > fx["max_attn"][0][1]


@pytest.mark.parametrize("name", NAMES)
def test_seeded_construction_matches_reference_digests(name):
    fx = _load(name)
    cfg = mince_cfg(fx)
    torch.manual_seed(fx["seed"])
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    init = S.SegtranInitWeights(cfg)
    enc.apply(init.init_weights)
    enc.apply(init.tie_qk)
    enc.apply(init.add_identity_bias)
    ours = enc.state_dict()
    ref = {k: v for k, v in fx["init_digests"].items() if ".pos_coder.all_" not in k}
    assert sorted(ours) == sorted(ref)
    for k, v in ours.items():
        assert _digest(v) == ref[k], k
    # mince layers are not CrossAttFeatTrans: query and key stay untied
    for layer in enc.translayers:
        assert layer.key.weight is not layer.query.weight


def test_reference_state_dict_with_index_buffers_loads_strictly():
    fx = _load("mince2d")
    assert any(".pos_coder.all_" in k for k in fx["state_dict"])
    enc = S.SegtranFusionEncoder(mince_cfg(fx), "Fusion")
    enc.load_state_dict(fx["state_dict"], strict=True)
    for s in range(3):
        key = "pos_code_layers.%d.pos_coder.biases" % s
        assert torch.equal(enc.pos_code_layers[s].pos_coder.biases.detach(), fx["state_dict"][key])
