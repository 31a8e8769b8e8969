"""The evaluation metrics on the GPU (segtran_b200.metrics, csrc/sx_metrics.cu) against the reference's own
calculate_metric_percase (fixture), the medpy restatement at BraTS size (fixture of seeds, digests and metrics) and the
pure-torch brute-force definition.  dc, jc, hd and hd95 must be equal; asd within 1e-12 relative (an fp64 sum in
another order).  Needs neither scipy nor the reference."""
import numpy as np
import pytest
import torch

from oracle import metric_oracle as MO
from segtran_b200 import _lib
from segtran_b200 import metrics as SM
from tests.helpers import load_golden

pytestmark = pytest.mark.gpu


def _compare(metric, valid, want_metric, want_valid):
    want_metric = np.asarray(want_metric)
    assert np.array_equal(valid, np.asarray(want_valid))
    assert np.array_equal(metric[:, :3], want_metric[:, :3]), (metric, want_metric)
    np.testing.assert_allclose(metric[:, 3], want_metric[:, 3], rtol=1e-12, atol=0)


@pytest.mark.parametrize("case", ["brats", "empty", "soft", "argmax"])
def test_percase_matches_reference_fixture(case):
    c = load_golden("metrics_percase")["cases"][case]
    pred = c["pred"].long() if c["kind"] == "long" else c["pred"].float()
    gt = c["gt"].long() if c["kind"] == "long" else c["gt"].float()
    metric, valid = SM.calculate_metric_percase(pred.cuda(), gt.cuda(), c["K"])
    assert metric.dtype == np.float64 and metric.shape == (c["K"] - 1, 4)
    _compare(metric, valid, c["metric"].numpy(), c["valid"].numpy())


@pytest.mark.parametrize("dtype", [torch.uint8, torch.bool])
def test_percase_accepts_uint8_and_bool(dtype):
    c = load_golden("metrics_percase")["cases"]["brats"]
    metric, valid = SM.calculate_metric_percase(c["pred"].to(dtype).cuda(), c["gt"].to(dtype).cuda(), 4)
    _compare(metric, valid, c["metric"].numpy(), c["valid"].numpy())


def test_fullsize_cases_match_restatement_with_hd95():
    fx = load_golden("metrics_fullsize")
    for c in fx["cases"]:
        p, g = MO.brats_like_case(c["seed"], tuple(c["shape"]), c["K"], empty=c["empty"])
        assert MO.sha256(p) == c["sha_pred"] and MO.sha256(g) == c["sha_gt"], "generator drifted for seed %d" % c["seed"]
        pc, gc = p.float().cuda(), g.float().cuda()
        metric, valid = SM.calculate_metric_percase(pc, gc, c["K"], hd95=True)
        _compare(metric, valid, c["metric"].numpy(), c["valid"].numpy())
        m0, v0 = SM.calculate_metric_percase(pc, gc, c["K"])
        want0 = c["metric"].numpy().copy()
        want0[:, 2] = 0
        _compare(m0, v0, want0, c["valid"].numpy())


def test_medpy_named_functions_match_brute_force():
    for a, b in MO.small_volumes(0) + MO.small_volumes(1):
        bf = MO.brute_metrics(a, b)
        ac, bc = a.cuda(), b.cuda()
        shape = tuple(a.shape)
        assert SM.dc(ac, bc) == bf["dc"], shape
        assert SM.jc(ac, bc) == bf["jc"], shape
        assert SM.hd(ac, bc) == bf["hd"], shape
        assert SM.hd95(ac, bc) == bf["hd95"], shape
        assert SM.asd(ac, bc) == pytest.approx(bf["asd"], rel=1e-12, abs=0), shape
        assert SM.assd(ac, bc) == pytest.approx(bf["assd"], rel=1e-12, abs=0), shape


def test_non_binary_operands_are_cast_to_bool():
    a = torch.zeros(9, 8, 7, device="cuda")
    b = torch.zeros(9, 8, 7, device="cuda")
    a[2:6, 2:5, 1:4] = 0.25                                  # non-zero: foreground for medpy's bool cast
    b[3:7, 2:6, 2:5] = 3.0
    bf = MO.brute_metrics(a.cpu() != 0, b.cpu() != 0)
    assert SM.dc(a, b) == bf["dc"] and SM.hd95(a, b) == bf["hd95"]


def test_two_calls_give_identical_bits():
    p, g = MO.brats_like_case(11, (96, 80, 64))
    pc, gc = p.cuda(), g.cuda()
    m1, v1 = SM.calculate_metric_percase(pc, gc, 4, hd95=True)
    m2, v2 = SM.calculate_metric_percase(pc, gc, 4, hd95=True)
    assert m1.tobytes() == m2.tobytes() and v1.tobytes() == v2.tobytes()


def test_errors():
    a = torch.zeros(6, 6, 6, device="cuda")
    a[1:3, 1:3, 1:3] = 1
    with pytest.raises(_lib.SxError):
        SM.asd(a.cpu(), a.cpu())
    with pytest.raises(NotImplementedError):
        SM.hd95(a, a, voxelspacing=(1.0, 1.0, 2.0))
    with pytest.raises(NotImplementedError):
        SM.asd(a, a, connectivity=2)
    with pytest.raises(ValueError):
        SM.asd(a[0, 0], a[0, 0])
    z = torch.zeros_like(a)
    for fn in (SM.asd, SM.hd95):
        with pytest.raises(RuntimeError, match="first"):
            fn(z, a)
        with pytest.raises(RuntimeError, match="second"):
            fn(a, z)
    assert SM.dc(z, z) == 0.0
