"""CPU checks of the positional-code ablations against fixtures made by the reference (oracle/gen_posbias_golden.py):
the float64 oracle reproduces the reference's outputs and gradients, seeded construction gives the reference's initial
parameters bit for bit, and a reference state_dict with its index buffers loads strictly."""
import hashlib
import os

import pytest
import torch

import segtran_b200.networks.segtran_shared as S
from oracle import posbias_oracle as PO
from tests.helpers import encoder_config

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["posbias3d", "posbias2d", "posbias_clamp", "posnone_sq"]


def _load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def _cfg(fx):
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"], num_attractors=fx["num_attractors"],
                         pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"])
    cfg.use_squeezed_transformer = fx["use_squeezed_transformer"]
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
    # Q and K are tied (tie_qk 'shared'): the state_dict carries both names for one tensor, the oracle reads `query`
    p = {k: v.double().requires_grad_() for k, v in fx["state_dict"].items()
         if v.is_floating_point() and not (k.endswith("key.weight") or k.endswith("key.bias"))}
    x = fx["x"].double().requires_grad_()
    y = PO.fusion_encoder_pos(p, "", x, fx["vmask"], fx["dims"], fx["num_modes"], fx["pos_code_type"], grid=fx["grid"],
                              pos_bias_radius=fx["pos_bias_radius"], pos_code_weight=fx["pos_code_weight"],
                              use_squeezed_transformer=fx["use_squeezed_transformer"])
    ref = fx["out"].double()
    assert float((y.detach() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    (y * fx["G"].double()).sum().backward()
    gx = fx["grad_x"].double()
    assert float((x.grad - gx).abs().max()) <= 1e-4 * float(gx.abs().max())
    checked = 0
    for k, g in fx["grad_params"].items():
        g = g.double()
        assert p[k].grad is not None, k
        assert float((p[k].grad - g).abs().max()) <= 1e-4 * float(g.abs().max()) + 1e-5, k     # floor: feat2score.bias grads are 0 up to fp32 noise
        checked += 1
    assert checked >= 10
    if fx["pos_code_type"] == "bias":
        assert "pos_code_layer.pos_coder.biases" in fx["grad_params"]


@pytest.mark.parametrize("name", NAMES)
def test_seeded_construction_matches_reference_digests(name):
    fx = _load(name)
    cfg = _cfg(fx)
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
    if fx["pos_code_type"] == "bias":
        idx = [k for k in fx["init_digests"] if ".pos_coder.all_" in k]
        assert len(idx) == 2 * fx["pos_dim"]


def test_reference_state_dict_with_index_buffers_loads_strictly():
    fx = _load("posbias2d")
    assert any(".pos_coder.all_" in k for k in fx["state_dict"])
    enc = S.SegtranFusionEncoder(_cfg(fx), "Fusion")
    enc.apply(S.SegtranInitWeights(_cfg(fx)).tie_qk)
    enc.load_state_dict(fx["state_dict"], strict=True)
    assert torch.equal(enc.pos_code_layer.pos_coder.biases.detach(), fx["state_dict"]["pos_code_layer.pos_coder.biases"])
