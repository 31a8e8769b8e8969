"""CPU checks of the attention-consistency losses: the float64 oracle reproduces the reference's losses and score
gradients on the fixtures of oracle/gen_consist_golden.py, and the drop-in functions refuse bad inputs before any
device work."""
import os

import pytest
import torch

from oracle import consist_oracle as CO
from segtran_b200 import train

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NAMES = ["consist3d_pair", "consist3d_pair2", "consist2d_pair", "consist2d_pair_cap", "consist2d_dense", "consist3d_dense"]


def _load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), map_location="cpu", weights_only=False)


def _entries(fx, dtype):
    return [[t.to(dtype).clone().requires_grad_() for t in e] if isinstance(e, list) else
            e.to(dtype).clone().requires_grad_() for e in fx["entries"]]


def _flat(entries):
    return [t for e in entries for t in (e if isinstance(e, list) else [e])]


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fixture(name):
    fx = _load(name)
    ent = _entries(fx, torch.float64)
    fun = CO.consist_loss3d if fx["three_d"] else CO.consist_loss2d
    kw = {} if fx["only_first_layer"] is None else {"only_first_layer": fx["only_first_layer"]}
    loss = fun(ent, torch.Size(fx["grid"]), fx["mask"].double(), **kw)
    loss.backward()
    assert abs(float(loss) - float(fx["loss"])) <= 1e-5 * max(1.0, abs(float(fx["loss"])))
    for t, g in zip(_flat(ent), fx["grads"]):
        got = torch.zeros_like(t) if t.grad is None else t.grad
        scale = max(float(g.abs().max()), 1e-12)
        assert float((got - g.double()).abs().max()) <= 1e-4 * scale


def test_cap_fixture_is_capped():
    assert float(_load("consist2d_pair_cap")["loss"]) == 1.0
    assert float(_load("consist2d_pair")["loss"]) < 1.0


def _pair(B, N, A):
    return [[torch.randn(B, 1, A, N), torch.randn(B, 1, N, A)]]


def test_refuses_batch_mismatch():
    with pytest.raises(ValueError, match="batch"):
        train.attn_consist_loss3d(_pair(2, 24, 8), (2, 3, 4), torch.zeros(3, 2, 6, 8, 4))


def test_refuses_token_count_mismatch():
    with pytest.raises(ValueError, match="tokens"):
        train.attn_consist_loss3d(_pair(2, 25, 8), (2, 3, 4), torch.zeros(2, 2, 6, 8, 4))
    with pytest.raises(ValueError, match="tokens"):
        train.attn_consist_loss2d([torch.randn(2, 1, 12, 13)], (3, 4), torch.zeros(2, 2, 6, 8))


def test_refuses_more_than_16_mask_channels():
    with pytest.raises(ValueError, match="16"):
        train.attn_consist_loss2d(_pair(2, 12, 8), (3, 4), torch.zeros(2, 17, 6, 8))


def test_refuses_wrong_mask_rank():
    with pytest.raises(ValueError):
        train.attn_consist_loss3d(_pair(2, 12, 8), (3, 4), torch.zeros(2, 2, 6, 8))


@pytest.mark.parametrize("name", ["consist_enc3d", "consist_enc2d_dense"])
def test_encoder_fixture_loads_strictly(name):
    """The reference encoder's state_dict with --attnconsist (attn_scaler included) loads into this build's encoder."""
    import segtran_b200.networks.segtran_shared as S
    from tests.helpers import encoder_config
    fx = _load(name)
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"], num_attractors=fx["num_attractors"],
                         pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"])
    cfg.use_squeezed_transformer = fx["use_squeezed_transformer"]
    cfg.use_attn_consist_loss = True
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    enc.load_state_dict(fx["state_dict"], strict=True)
    assert any(k.startswith("attn_scaler") for k in fx["state_dict"])
