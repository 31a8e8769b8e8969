"""CPU checks of the multi-head ablation (--nosqueeze --multihead): the oracle reproduces the reference's outputs,
gradients and max_attn on the fixtures of oracle/gen_multihead_golden.py (float64 against the reference's float32), seeded construction gives the reference's initial
parameters bit for bit, reference state_dicts load strictly, and the combinations the reference cannot run are refused."""
import hashlib

import pytest
import torch
import torch.nn.functional as F

import segtran_b200.networks.segtran_shared as S
from oracle import consist_oracle as CO
from oracle import multihead_oracle as MH
from tests.helpers import encoder_config, load_golden

NAMES = ["multihead_2d", "multihead_3d_compress", "multihead_sharedout", "multihead_posbias", "multihead_posnone",
         "multihead_clamp", "multihead_consist", "multihead_d9"]


# (output, gradient) tolerances, max|a-b|/max|b|: the reference computes in float32; in multihead_clamp its scores reach
# ~7000, where one float32 ulp of a score is 5e-4
TOLS = {"multihead_clamp": (3e-5, 1e-3)}


def mh_cfg(fx):
    cfg = encoder_config(S.SegtranConfig, dims=fx["dims"], num_modes=fx["num_modes"], num_attractors=fx["num_attractors"],
                         pos_dim=fx["pos_dim"], qk_have_bias=fx["qk_have_bias"])
    cfg.use_squeezed_transformer = False
    cfg.ablate_multihead = True
    cfg.trans_output_type = fx["trans_output_type"]
    cfg.pos_code_type = fx["pos_code_type"]
    cfg.pos_bias_radius = fx["pos_bias_radius"]
    cfg.pos_code_weight = fx["pos_code_weight"]
    cfg.max_pos_size = tuple(fx["grid"])
    cfg.use_attn_consist_loss = fx["use_attn_consist_loss"]
    return cfg


def oracle_loss(fx, p, x):
    """The fixture's loss on the oracle: (out * G).sum(), or the attention-consistency loss of the kept scores."""
    stats = {}
    y = MH.fusion_encoder_multihead(p, "", x, fx["voxels_pos"].to(x.dtype), fx["vmask"], fx["dims"], fx["num_modes"],
                                    pos_code_type=fx["pos_code_type"], grid=fx["grid"],
                                    pos_bias_radius=fx["pos_bias_radius"], pos_code_weight=fx["pos_code_weight"],
                                    trans_output_type=fx["trans_output_type"], collect=stats)
    if fx["use_attn_consist_loss"]:
        ent = [F.conv2d(s, p["attn_scaler.weight"], p["attn_scaler.bias"]) for s in stats["scores"]]
        fun = CO.consist_loss3d if fx["three_d"] else CO.consist_loss2d
        return y, fun(ent, torch.Size(fx["grid"]), fx["seg_mask"].to(x.dtype)), stats
    return y, (y * fx["G"].to(x.dtype)).sum(), stats


def _digest(t):
    t = t.detach().cpu().contiguous()
    return tuple(t.shape), str(t.dtype), hashlib.sha256(t.numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_fixture(name):
    fx = load_golden(name)
    # the key projection is tied to the query's (tie_qk 'shared'): the oracle reads `query` for both
    p = {k: v.double().requires_grad_() for k, v in fx["state_dict"].items()
         if v.is_floating_point() and ".key." not in k}
    x = fx["x"].double().requires_grad_()
    y, loss, stats = oracle_loss(fx, p, x)
    out_tol, grad_tol = TOLS.get(name, (1e-6, 1e-5))
    ref = fx["out"].double()
    assert float((y.detach() - ref).abs().max()) <= out_tol * float(ref.abs().max())
    if fx["use_attn_consist_loss"]:
        assert abs(float(loss) - float(fx["loss"])) <= 1e-6 * abs(float(fx["loss"]))
    loss.backward()
    gx = fx["grad_x"].double()
    assert float((x.grad - gx).abs().max()) <= grad_tol * float(gx.abs().max())
    for k, g in fx["grad_params"].items():
        g = g.double()
        assert p[k].grad is not None, k
        assert float((p[k].grad - g).abs().max()) <= grad_tol * float(g.abs().max()) + 1e-9, k
    for ours, theirs in zip(stats["max_attn"], fx["max_attn"]):
        assert ours == pytest.approx(theirs, rel=1e-5, abs=1e-6)


def test_fixtures_cover_the_clamp_and_the_unaligned_heads():
    assert load_golden("multihead_clamp")["max_attn"][0] > 500
    fx = load_golden("multihead_d9")
    assert fx["dims"] == [36, 36] and fx["num_modes"] == 4                   # d = dh = 9
    assert load_golden("multihead_2d")["grid"] == [12, 12]                     # 144 keys: more than one key chunk


@pytest.mark.parametrize("name", NAMES)
def test_seeded_construction_matches_reference_digests(name):
    fx = load_golden(name)
    cfg = mh_cfg(fx)
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
    assert [t.config.num_modes for t in enc.translayers] == fx["layer_num_modes"] == [1] * len(enc.translayers)


@pytest.mark.parametrize("name", NAMES)
def test_reference_state_dict_loads_strictly(name):
    fx = load_golden(name)
    cfg = mh_cfg(fx)
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    enc.apply(S.SegtranInitWeights(cfg).tie_qk)
    enc.load_state_dict(fx["state_dict"], strict=True)


def test_state_dict_keys_and_shapes():
    for out_type in ("private", "shared"):
        cfg = encoder_config(S.SegtranConfig, dims=[64, 64, 32], num_modes=4, num_attractors=4, pos_dim=3)
        cfg.use_squeezed_transformer = False
        cfg.ablate_multihead = True
        cfg.trans_output_type = out_type
        sd = S.SegtranFusionEncoder(cfg, "Fusion").state_dict()
        pre = "translayers.1.out_trans."
        assert sd[pre + "first_linear.weight"].shape == (32, 64) and sd[pre + "first_linear.bias"].shape == (32,)
        assert sd[pre + "intermediate.shared_linear.weight"].shape == (32, 32)
        assert sd[pre + "intermediate.shared_linear.bias"].shape == (32,)
        if out_type == "private":
            assert sd[pre + "output.group_linear.weight"].shape == (32, 32, 1)
            assert sd[pre + "output.group_linear.bias"].shape == (32,)
        else:
            assert sd[pre + "output.shared_linear.weight"].shape == (32, 32)
        assert sd[pre + "output.resout_norm_layer.weight"].shape == (32,)
        keys = sorted(k[len("translayers.1."):] for k in sd if k.startswith("translayers.1."))
        other = "output.group_linear" if out_type == "private" else "output.shared_linear"
        want = ["key.bias", "key.weight", "query.bias", "query.weight"] + \
            ["out_trans." + n for n in ("first_linear.bias", "first_linear.weight", "intermediate.shared_linear.bias",
                                        "intermediate.shared_linear.weight", other + ".bias", other + ".weight",
                                        "output.resout_norm_layer.bias", "output.resout_norm_layer.weight")]
        assert keys == sorted(want)
        assert not any("feat_softaggr" in k or "first_norm_layer" in k for k in sd)


def test_num_modes_mutation_stays_on_the_layer_config():
    cfg = encoder_config(S.SegtranConfig, dims=[32, 32], num_modes=4, num_attractors=4, pos_dim=3)
    cfg.use_squeezed_transformer = False
    cfg.ablate_multihead = True
    cfg.use_attn_consist_loss = True
    enc = S.SegtranFusionEncoder(cfg, "Fusion")
    layer = enc.translayers[0]
    assert cfg.num_modes == 4 and layer.num_modes == 4 and layer.out_trans.num_modes == 4
    assert layer.config.num_modes == 1 and layer.out_trans.config is layer.config
    assert layer.out_trans.intermediate.num_modes == 1
    assert enc.attn_scaler.weight.shape == (1, 4, 1, 1)
    assert isinstance(layer.out_trans, S.MultiHeadFeatTrans) and not isinstance(layer.out_trans, S.ExpandedFeatTrans)


def test_refused_combinations():
    cfg = encoder_config(S.SegtranConfig, dims=[32, 32], num_modes=4, num_attractors=4, pos_dim=3)
    cfg.ablate_multihead = True
    with pytest.raises(NotImplementedError, match="segtran_ablation.py:239"):     # squeezed: the reference crashes
        S.SegtranFusionEncoder(cfg, "Fusion")
    cfg.use_squeezed_transformer = False
    cfg.use_mince_transformer = True
    cfg.mince_scales, cfg.mince_channel_props = [1, 2], [1, 1]
    with pytest.raises(NotImplementedError):
        S.SegtranFusionEncoder(cfg, "Fusion")
    for mid in ("private", None):
        cfg = encoder_config(S.SegtranConfig, dims=[32, 32], num_modes=4, num_attractors=4, pos_dim=3)
        cfg.use_squeezed_transformer = False
        cfg.ablate_multihead = True
        cfg.mid_type = mid
        with pytest.raises(NotImplementedError):
            S.SegtranFusionEncoder(cfg, "Fusion")


def test_feat_dim_not_divisible_by_heads_raises_value_error():
    cfg = encoder_config(S.SegtranConfig, dims=[32, 30], num_modes=4, num_attractors=4, pos_dim=3)
    cfg.use_squeezed_transformer = False
    cfg.ablate_multihead = True
    with pytest.raises(ValueError):
        S.SegtranFusionEncoder(cfg, "Fusion")
