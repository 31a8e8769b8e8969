"""CPU checks of the evaluation metrics: the scipy restatement of medpy's functions (oracle/metric_oracle.py) against a
pure-torch brute-force definition, the restatement of calculate_metric_percase against the fixture the reference's own
function produced (oracle/gen_metric_golden.py), and the argument checks of segtran_b200.metrics that need no device."""
import numpy as np
import pytest
import torch

from oracle import metric_oracle as MO
from segtran_b200 import _lib
from segtran_b200 import metrics as SM
from tests.helpers import load_golden


@pytest.mark.parametrize("seed", [0, 1])
def test_restatement_matches_brute_force(seed):
    for a, b in MO.small_volumes(seed):
        bf = MO.brute_metrics(a, b)
        an, bn = a.numpy(), b.numpy()
        assert MO.dc(an, bn) == bf["dc"]
        assert MO.jc(an, bn) == bf["jc"]
        assert MO.hd(an, bn) == bf["hd"], tuple(a.shape)
        assert MO.hd95(an, bn) == bf["hd95"], tuple(a.shape)
        assert MO.asd(an, bn) == pytest.approx(bf["asd"], rel=1e-12, abs=0)
        assert MO.assd(an, bn) == pytest.approx(bf["assd"], rel=1e-12, abs=0)


def test_brute_force_border_and_percentile_by_hand():
    x = torch.zeros(5, 5, dtype=torch.bool)
    x[1:4, 1:4] = True
    want = x.clone()
    want[2, 2] = False
    assert torch.equal(MO.brute_border(x), want)
    assert MO.brute_border(torch.ones(1, 7, dtype=torch.bool)).all()          # an extent of 1 erodes everything in 2-D
    assert MO.brute_percentile95(torch.tensor([0., 1., 2., 3.])) == np.percentile([0., 1., 2., 3.], 95)
    vals = torch.from_numpy(np.sqrt(np.random.default_rng(0).integers(0, 50, 37).astype(np.float64)))
    assert MO.brute_percentile95(vals) == np.percentile(vals.numpy(), 95)


def test_empty_masks_raise_in_restatement():
    z, o = np.zeros((4, 4), bool), np.ones((4, 4), bool)
    with pytest.raises(RuntimeError):
        MO.asd(z, o)
    with pytest.raises(RuntimeError):
        MO.hd95(o, z)
    assert MO.dc(z, z) == 0.0


@pytest.mark.parametrize("case", ["brats", "empty", "soft", "argmax"])
def test_restated_percase_matches_reference_fixture(case):
    c = load_golden("metrics_percase")["cases"][case]
    pred = c["pred"].long() if c["kind"] == "long" else c["pred"].float()
    gt = c["gt"].long() if c["kind"] == "long" else c["gt"].float()
    metric, valid = MO.calculate_metric_percase(pred, gt, c["K"])
    assert np.array_equal(valid, c["valid"].numpy())
    assert np.array_equal(metric[:, :3], c["metric"].numpy()[:, :3])
    np.testing.assert_allclose(metric[:, 3], c["metric"].numpy()[:, 3], rtol=1e-12, atol=0)


def test_fullsize_fixture_is_small_and_complete():
    fx = load_golden("metrics_fullsize")
    assert len(fx["cases"]) >= 2
    for c in fx["cases"]:
        assert tuple(c["shape"]) == (240, 240, 155) and c["K"] == 4
        assert len(c["sha_pred"]) == 64 and len(c["sha_gt"]) == 64
        assert c["metric"].shape == (3, 4) and c["valid"].shape == (3, 4)


def test_generator_is_seeded_and_shaped():
    p1, g1 = MO.brats_like_case(5, (20, 18, 11))
    p2, g2 = MO.brats_like_case(5, (20, 18, 11))
    assert torch.equal(p1, p2) and torch.equal(g1, g2)
    assert p1.shape == (4, 20, 18, 11) and p1.dtype == torch.uint8
    assert g1[3, 0].any()                                              # the last class touches the first face
    p3, _ = MO.brats_like_case(5, (20, 18, 11), empty=("pred", 2))
    assert not p3[2].any()


def test_argument_checks_without_a_device():
    a = torch.zeros(4, 4)
    with pytest.raises(NotImplementedError):
        SM.asd(a, a, voxelspacing=(1.0, 2.0))
    with pytest.raises(NotImplementedError):
        SM.hd95(a, a, connectivity=2)
    with pytest.raises(_lib.SxError):                                  # no CPU fallback
        SM.dc(a, a)
    with pytest.raises(_lib.SxError):
        SM.calculate_metric_percase(torch.zeros(4, 3, 3, 3), torch.zeros(4, 3, 3, 3), 4)


def test_metric_entry_points_are_bound():
    for name in ("sx_mask_counts", "sx_surface", "sx_edt_sq", "sx_surface_hist", "sx_surface_stats"):
        assert name in _lib._PROTOS and name in _lib.EXPORTS
