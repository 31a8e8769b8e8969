"""2-D sliding-window inference (segtran_b200.inference.test_single_batch) and per-image evaluation
(segtran_b200.metrics.calc_batch_metric / calc_vcdr, csrc/sx_eval2d.cu) against the reference-generated fixtures
(tests/golden/eval2d.pt) and, at the REFUGE size, against the oracle run on the same GPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import eval2d_oracle as E
from tests.helpers import AffinePickNet, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return load_golden("eval2d")


def _check_sw(hard, soft, ref_hard, ref_soft):
    hard, soft = hard.cpu(), soft.cpu()
    assert hard.dtype == torch.int32 and soft.dtype == torch.float32
    assert hard.shape == ref_hard.shape and soft.shape == ref_soft.shape
    assert float((soft - ref_soft).abs().max()) < 2e-6
    sure = (ref_soft - 0.5).abs() > 1e-5                   # away from the threshold the hard maps must be identical
    sure[:, 0] = sure[:, 1:].all(dim=1)
    assert torch.equal(hard[sure], ref_hard[sure])
    assert float(sure.float().mean()) > 0.999


def test_sliding_window_matches_reference_fixtures(fx):
    from segtran_b200.inference import test_single_batch
    for key, c in fx["sw"].items():
        net = AffinePickNet(c["a"], c["b"], c["ch"]).cuda()
        hard, soft = test_single_batch(net, c["image"].cuda(), c["orig"], c["patch"], c["stride"], "fundus", c["K"],
                                       "segtran")
        assert hard.shape[2:] == c["image"].shape[2:], key          # padding cropped away
        _check_sw(hard, soft, c["hard"], c["soft"])


def test_sliding_window_pranet_and_nnunet_outputs():
    from segtran_b200.inference import test_single_batch
    torch.manual_seed(5)
    image = torch.randn(2, 3, 30, 44) * 2
    inner = AffinePickNet([1.3, 0.8], [0.2, -0.1], [1, 2])

    class PraNetLike(torch.nn.Module):                    # four side outputs; [3] lacks the background channel
        def forward(self, x):
            y = inner(x)
            return (y * 2, y * 3, y * 4, y)

    class NnUNetLike(torch.nn.Module):                    # deep supervision: the full-resolution output first
        def forward(self, x):
            y = AffinePickNet([1.1, 0.9, 1.4], [0., 0.1, -0.2], [0, 1, 2])(x)
            return [y, y[:, :, ::2, ::2]]

    for net, mt, K in ((PraNetLike(), "pranet", 3), (NnUNetLike(), "nnunet", 3)):
        args = ((32, 32), (16, 16), (16, 12), "fundus", K, mt)
        ref_hard, ref_soft = E.test_single_batch(net, image, *args)
        hard, soft = test_single_batch(net, image.cuda(), *args)
        _check_sw(hard, soft, ref_hard, ref_soft)


def _cuda(x):
    return [t.cuda() for t in x] if isinstance(x, list) else x.cuda()


def _decided(pred, gt, K, vcdr):
    """[B, K-1+vcdr] bool: True where the column's hard masks cannot depend on the last bits of the resize — no value of
    its classes in the prediction resized to the ground truth's size (on the host, as the reference does) lies within
    1e-5 of the threshold.  The vCDR column depends on classes 1 and 2."""
    out = []
    for p, g in zip(pred, gt):
        p = p.cpu()
        if tuple(p.shape[1:]) == tuple(g.shape[1:]):
            out.append([True] * (K - 1 + vcdr))
            continue
        r = F.interpolate(p.unsqueeze(0), size=g.shape[1:], mode='bilinear', align_corners=False)[0]
        far = [bool(((r[c] - 0.5).abs() > 1e-5).all()) for c in range(1, K)]
        out.append(far + ([far[0] and far[1]] if vcdr else []))
    return np.array(out, dtype=bool)


def test_batch_metric_matches_reference_fixtures(fx):
    from segtran_b200.metrics import calc_batch_metric
    checked = total = 0
    for key, c in fx["metric"].items():
        for vcdr, ref in c["metric"].items():
            ok = _decided(c["pred"], c["gt"], c["K"], vcdr)
            out = calc_batch_metric(_cuda(c["pred"]), _cuda(c["gt"]), c["K"], do_calc_vcdr_error=vcdr)
            assert out.dtype == np.float64 and out.shape == tuple(ref.shape), key
            assert np.array_equal(out[ok], ref.numpy()[ok]), (key, vcdr, out, ref)
            checked, total = checked + int(ok.sum()), total + ok.size
            if key == "same_size":
                assert ok.all()
    assert checked >= 0.8 * total, (checked, total)


def test_batch_metric_float_and_uint8_ground_truth_agree(fx):
    from segtran_b200.metrics import calc_batch_metric
    c = fx["metric"]["ellipse"]
    a = calc_batch_metric(c["pred"].cuda(), c["gt"].cuda(), 3, do_calc_vcdr_error=True)
    b = calc_batch_metric(c["pred"].cuda(), c["gt"].float().cuda(), 3, do_calc_vcdr_error=True)
    assert np.array_equal(a, b)


def test_calc_vcdr_matches_oracle(fx):
    from segtran_b200.metrics import calc_vcdr
    for key in ("ellipse", "edges", "same_size"):
        c = fx["metric"][key]
        gt = c["gt"].float()
        for b in range(gt.shape[0]):
            hard = E.harden_segmap2d(c["pred"][b])
            for m in (gt[b], hard, c["pred"][b]):
                v = calc_vcdr(m.cuda())
                ref = E.calc_vcdr(m)
                assert v.is_cuda and v.dim() == 0 and v.dtype == ref.dtype == torch.float32
                assert torch.equal(v.cpu(), ref), (key, b, float(v), float(ref))


def test_non_binary_ground_truth_raises(fx):
    from segtran_b200.metrics import calc_batch_metric
    c = fx["metric"]["ellipse"]
    gt = c["gt"].float()
    gt[1, 2, 10, 10] = 0.5
    with pytest.raises(ValueError, match="binary"):
        calc_batch_metric(c["pred"].cuda(), gt.cuda(), 3)


def test_deterministic(fx):
    from segtran_b200.inference import test_single_batch
    from segtran_b200.metrics import calc_batch_metric
    c = fx["sw"]["polyp_overlap"]
    net = AffinePickNet(c["a"], c["b"], c["ch"]).cuda()
    runs = [test_single_batch(net, c["image"].cuda(), c["orig"], c["patch"], c["stride"], "polyp", c["K"], "segtran")
            for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    m = fx["metric"]["ellipse"]
    a = calc_batch_metric(m["pred"].cuda(), m["gt"].cuda(), 3, do_calc_vcdr_error=True)
    b = calc_batch_metric(m["pred"].cuda(), m["gt"].cuda(), 3, do_calc_vcdr_error=True)
    assert a.tobytes() == b.tobytes()


def test_cpu_tensors_raise(fx):
    from segtran_b200 import _lib
    from segtran_b200.inference import test_single_batch
    from segtran_b200.metrics import calc_batch_metric, calc_vcdr
    c = fx["sw"]["single_x2"]
    with pytest.raises(_lib.SxError):
        test_single_batch(AffinePickNet(c["a"], c["b"], c["ch"]), c["image"], c["orig"], c["patch"], c["stride"],
                          "fundus", c["K"], "segtran")
    m = fx["metric"]["ellipse"]
    with pytest.raises(_lib.SxError):
        calc_batch_metric(m["pred"], m["gt"], 3)
    with pytest.raises(_lib.SxError):
        calc_vcdr(m["gt"][0].float())


def test_refuge_size_against_oracle_on_gpu():
    """B=4 fundus images at 576x576, one window resized to 288 and its scores upsampled x2 (the REFUGE default), then
    the metrics with vCDR against 576x576 ground truths, both from our soft maps and from ones at half size."""
    from segtran_b200.inference import test_single_batch
    from segtran_b200.metrics import calc_batch_metric
    torch.manual_seed(17)
    image = (torch.randn(4, 3, 576, 576) * 2).cuda()
    net = AffinePickNet([1.2, 1.6, 2.0], [-0.4, -0.1, 0.2], [0, 1, 2]).cuda()
    args = ((576, 576), (288, 288), (288, 288), "fundus", 3, "segtran")
    ref_hard, ref_soft = E.test_single_batch(net, image, *args)
    hard, soft = test_single_batch(net, image, *args)
    _check_sw(hard, soft, ref_hard.cpu(), ref_soft.cpu())

    gt = E.fundus_like_gt(4, 576, 576, seed=71).cuda()
    pred = E.soft_from_gt(E.fundus_like_gt(4, 576, 576, 71, jitter=0.3, jitter_seed=72), 576, 576, seed=73).cuda()
    half = E.soft_from_gt(E.fundus_like_gt(4, 576, 576, 71, jitter=0.3, jitter_seed=74), 288, 288, seed=75).cuda()
    for p in (pred, half):
        for vcdr in (False, True):
            out = calc_batch_metric(p, gt, 3, do_calc_vcdr_error=vcdr)
            ref = E.calc_batch_metric(p, gt, 3, do_calc_vcdr_error=vcdr)
            ok = _decided(p, gt, 3, vcdr)
            assert np.array_equal(out[ok], ref[ok]), (vcdr, out, ref)
            assert ok.all() or p is half
