"""Mirror test-time augmentation (``mirror_axes`` of segtran_b200.inference) on the CPU: the stock-PyTorch TTA oracle
(oracle/tta_oracle.py) against fixtures made from the reference's own sliding-window functions
(tests/golden/tta_*.pt, oracle/gen_tta_golden.py), the C-ABI declarations, and the argument errors."""
import ctypes
import glob
import os

import pytest
import torch

from oracle import tta_oracle as IO
from tests.helpers import GOLDEN, AffinePickNet, load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TTA = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(GOLDEN, "tta_*.pt")))


def sure_mask(ref_soft, ref_hard, kind):
    """Where the hard masks must agree: away from the BraTS threshold / from an arg-max or harden_segmap2d tie."""
    if kind == "tta3d" and ref_hard.dim() == ref_soft.dim():           # BraTS: [K,H,W,D] masks
        sure = (ref_soft - 0.5).abs() > 1e-5
        sure[0] = sure[1:].all(dim=0)
        return sure
    if kind == "tta3d":
        top2 = ref_soft.topk(2, dim=0).values
        return (top2[0] - top2[1]) > 1e-5
    sure = (ref_soft - 0.5).abs() > 1e-5
    sure[:, 0] = sure[:, 1:].all(dim=1)
    return sure


def run_oracle(fx, net, image):
    if fx["kind"] == "tta3d":
        return IO.test_single_case_tta(net, image, fx["orig_patch"], fx["input_patch"], fx["batch_size"], fx["stride_xy"],
                                       fx["stride_z"], fx["task"], "segtran", fx["K"], fx["mirror_axes"])
    return IO.test_single_batch_tta(net, image, fx["orig"], fx["patch"], fx["stride"], "fundus", fx["K"], "segtran",
                                    fx["mirror_axes"])


def test_fixtures_cover_the_cases():
    assert len(TTA) == 5
    fxs = {n: load_golden(n) for n in TTA}
    three = [f for f in fxs.values() if f["kind"] == "tta3d"]
    assert {len(f["mirror_axes"]) for f in three} == {1, 2, 3}
    assert {f["task"] for f in three} == {"brats", "other"} and any(f["K"] == 2 for f in three)
    assert any(tuple(f["image"].shape[1:]) < tuple(f["orig_patch"]) for f in three)              # a padded volume
    two = [f for f in fxs.values() if f["kind"] == "tta2d"]
    assert {f["patch"] == f["orig"] for f in two} == {True, False}
    assert any(f["image"].shape[2] < f["orig"][0] for f in two)                                  # a padded batch


@pytest.mark.parametrize("name", TTA)
def test_tta_oracle_matches_reference_fixtures(name):
    fx = load_golden(name)
    hard, soft = run_oracle(fx, IO.AsymNet(**fx["net"]), fx["image"])
    assert soft.shape == fx["soft"].shape and hard.shape == fx["hard"].shape and hard.dtype == fx["hard"].dtype
    assert (soft - fx["soft"]).abs().max() < 1e-6
    sure = sure_mask(fx["soft"], fx["hard"], fx["kind"])
    assert float(sure.float().mean()) > 0.99
    assert torch.equal(hard[sure], fx["hard"][sure])


@pytest.mark.parametrize("name", TTA)
def test_the_fixture_net_is_not_mirror_equivariant(name):
    """TTA changes the fixtures' output: the plain sliding window differs from the mirrored average."""
    fx = load_golden(name)
    _, soft = run_oracle(dict(fx, mirror_axes=()), IO.AsymNet(**fx["net"]), fx["image"])
    assert (soft - fx["soft"]).abs().max() > 1e-2


def test_no_mirror_axes_is_the_plain_oracle():
    fx = load_golden("infer_sw")
    c = fx["cases"]["brats_resized"]
    net = AffinePickNet(c["a"], c["b"], c["ch"])
    args = (c["orig_patch"], c["input_patch"], c["batch_size"], c["stride_xy"], c["stride_z"], c["task"], "segtran", c["K"])
    hard, soft = IO.test_single_case_tta(net, c["image"], *args, ())
    assert torch.equal(soft, c["soft"]) and torch.equal(hard, c["hard"])


def test_header_declares_the_mirror_entry_points():
    from segtran_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "segtran_b200.h")).read()
    assert "int sx_sw_gather(" in hdr and "sx_sw_gather" in _lib.EXPORTS
    assert len(_lib._PROTOS["sx_sw_accumulate"]) == 16 and len(_lib._PROTOS["sx_sw2d_accumulate"]) == 16
    assert len(_lib._PROTOS["sx_sw_gather"]) == 14
    readme = open(os.path.join(ROOT, "README.md")).read()
    assert "(71 entry points)" in readme


def _refused(name, *args):
    from segtran_b200 import _lib as L
    with pytest.raises(L.SxError) as e:
        L.call(name, *args)
    return str(e.value)


def test_kernels_refuse_bad_masks_and_windows_before_any_launch():
    org = (ctypes.c_int32 * 6)(0, 0, 0, 2, 2, 2)
    assert "mirror mask 8" in _refused("sx_sw_gather", 0, 1, 2, 4, 4, 4, org, 2, 2, 2, 2, 8, 0, None)
    assert "mirror mask -1" in _refused("sx_sw_gather", 0, 1, 2, 4, 4, 4, org, 2, 2, 2, 2, -1, 0, None)
    assert "window 1" in _refused("sx_sw_gather", 0, 1, 2, 4, 4, 4, org, 2, 3, 3, 3, 1, 0, None)
    assert "empty" in _refused("sx_sw_gather", 0, 1, 2, 4, 4, 4, None, 2, 2, 2, 2, 1, 0, None)
    assert "mirror mask 8" in _refused("sx_sw_accumulate", 0, 4, 2, 2, 2, 0, 0, 4, 4, 4, 0, 0, 0, 8, None, None)
    assert "mirror mask 4" in _refused("sx_sw2d_accumulate", 0, 1, 3, 2, 2, 4, 4, 0, 0, 8, 8, 0, 0, 4, None, None)


@pytest.mark.parametrize("axes", [(0, 0), (3,), (-1,), (0, 1, 2, 0), 0, "01", {0, 1}, (True,), (0.0,), None])
def test_bad_mirror_axes_raise_value_error_before_any_launch(axes):
    from segtran_b200.inference import test_single_batch, test_single_case
    net = AffinePickNet([1.0, 1.0], [0.0, 0.0], [0, 0])
    with pytest.raises(ValueError):
        test_single_case(net, torch.zeros(1, 8, 8, 8), (8, 8, 8), (8, 8, 8), 1, 8, 8, "other", "segtran", 2,
                         mirror_axes=axes)
    with pytest.raises(ValueError):
        test_single_batch(net, torch.zeros(1, 1, 8, 8), (8, 8), (8, 8), (8, 8), "fundus", 2, "segtran",
                          mirror_axes=axes if axes != (3,) else (2,))


def test_valid_mirror_axes_still_need_a_gpu():
    from segtran_b200 import _lib as L
    from segtran_b200.inference import test_single_batch, test_single_case
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    net = AffinePickNet([1.0, 1.0], [0.0, 0.0], [0, 0])
    with pytest.raises(L.SxError):
        test_single_case(net, torch.zeros(1, 8, 8, 8), (8, 8, 8), (8, 8, 8), 1, 8, 8, "other", "segtran", 2,
                         mirror_axes=[2, 0])
    with pytest.raises(L.SxError):
        test_single_batch(net, torch.zeros(1, 1, 8, 8), (8, 8), (8, 8), (8, 8), "fundus", 2, "segtran", mirror_axes=(1,))


def test_variant_masks_follow_the_bit_order():
    from segtran_b200.inference import _mirror_masks
    assert _mirror_masks((), 3, "t") == [0]
    assert _mirror_masks((2, 0), 3, "t") == [0, 4, 1, 5]
    assert _mirror_masks((1, 0), 2, "t") == [0, 2, 1, 3]
    assert _mirror_masks((0, 1, 2), 3, "t") == list(range(8))
    assert IO.mirror_dims((2, 0), 2) == [[], [4], [2], [4, 2]]
