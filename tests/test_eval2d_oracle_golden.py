"""The 2-D evaluation oracle (oracle/eval2d_oracle.py) against fixtures made by the reference's own test_util2d functions
(tests/golden/eval2d.pt, oracle/gen_eval2d_golden.py), and the host side of segtran_b200.metrics' 2-D drop-ins: the fp32
values it derives from integer counts, and the arguments it refuses."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import eval2d_oracle as E
from tests.helpers import AffinePickNet, load_golden


@pytest.fixture(scope="module")
def fx():
    return load_golden("eval2d")


def _gt_float(g):
    return [t.float() for t in g] if isinstance(g, list) else g.float()


def test_sliding_window_oracle_matches_reference_fixtures(fx):
    for key, c in fx["sw"].items():
        net = AffinePickNet(c["a"], c["b"], c["ch"])
        hard, soft = E.test_single_batch(net, c["image"], c["orig"], c["patch"], c["stride"], "fundus", c["K"], "segtran")
        assert soft.shape == c["soft"].shape and hard.dtype == c["hard"].dtype == torch.int32, key
        assert float((soft - c["soft"]).abs().max()) <= 1e-6, key
        assert torch.equal(hard, c["hard"]), key


def test_metric_oracle_matches_reference_fixtures(fx):
    for key, c in fx["metric"].items():
        for vcdr, ref in c["metric"].items():
            out = E.calc_batch_metric(c["pred"], _gt_float(c["gt"]), c["K"], do_calc_vcdr_error=vcdr)
            assert out.dtype == np.float64 and np.array_equal(out, ref.numpy()), (key, vcdr)


def _host_counts(pred_soft, gt, K):
    """what sx_eval2d_counts produces for one image, computed on the host from the oracle's resized, hardened prediction"""
    from segtran_b200.metrics import _eval2d_ld
    H = gt.shape[1]
    p = E.harden_segmap2d(F.interpolate(pred_soft.unsqueeze(0), size=gt.shape[1:], mode='bilinear',
                                        align_corners=False)[0]).bool()
    g = gt >= 0.5
    row = np.zeros(_eval2d_ld(K), dtype=np.int64)
    for c in range(1, K):
        row[3 * (c - 1):3 * c] = [int((p[c] & g[c]).sum()), int(p[c].sum()), int(g[c].sum())]
    for who, m in enumerate((p, g)):
        for c in (1, 2):
            if c >= K:
                continue
            occ = torch.nonzero(m[c].any(dim=1)).flatten()
            if len(occ):
                row[3 * (K - 1) + 4 * who + 2 * (c - 1):][:2] = [int(occ.max()) + 1, H - int(occ.min())]
    row[3 * (K - 1) + 8] = int(((gt[1:K] != 0) & (gt[1:K] != 1)).sum())
    return row


def test_values_from_counts_are_bit_identical_to_the_reference(fx):
    """The fp32 Dice / vCDR arithmetic of segtran_b200.metrics applied to exact counts reproduces every fixture."""
    from segtran_b200 import metrics as SM
    for key, c in fx["metric"].items():
        gts = _gt_float(c["gt"])
        counts = np.stack([_host_counts(p, g, c["K"]) for p, g in zip(c["pred"], gts)])
        for vcdr, ref in c["metric"].items():
            out = SM._batch_values(counts, c["K"], [g.shape[1] for g in gts], vcdr)
            assert np.array_equal(out, ref.numpy()), (key, vcdr, out, ref)


def test_non_binary_ground_truth_is_refused():
    from segtran_b200 import metrics as SM
    gt = E.fundus_like_gt(1, 20, 18, seed=3)[0]
    gt[1, 4, 5] = 0.5
    counts = _host_counts(E.soft_from_gt(gt.unsqueeze(0), 10, 9, seed=4)[0], gt, 3)[None]
    assert counts[0, -1] == 1
    with pytest.raises(ValueError, match="binary"):
        SM._batch_values(counts, 3, [20], False)


def test_vcdr_needs_three_classes():
    from segtran_b200 import metrics as SM
    p, g = torch.rand(2, 2, 8, 8), torch.zeros(2, 2, 8, 8)
    with pytest.raises(ValueError, match="num_classes >= 3"):
        SM.calc_batch_metric(p, g, 2, do_calc_vcdr_error=True)
