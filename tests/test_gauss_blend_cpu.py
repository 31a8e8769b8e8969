"""Gaussian window blending (``gaussian_sigma_scale`` of segtran_b200.inference) on the CPU: the stock-PyTorch oracle
(oracle/gauss_oracle.py) with unit weights against the reference-generated sliding-window fixtures, the per-axis weight
tables against a float64 restatement, the C-ABI declarations and refusals, and the argument errors."""
import os

import numpy as np
import pytest
import torch

from oracle import gauss_oracle as GO
from oracle import tta_oracle as TO
from tests.helpers import AffinePickNet, load_golden
from tests.test_tta_cpu import TTA, run_oracle, sure_mask

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_gauss(fx, net, image, weight):
    if fx["kind"] == "tta3d":
        return GO.test_single_case_gauss(net, image, fx["orig_patch"], fx["input_patch"], fx["batch_size"],
                                         fx["stride_xy"], fx["stride_z"], fx["task"], "segtran", fx["K"],
                                         fx["mirror_axes"], weight)
    return GO.test_single_batch_gauss(net, image, fx["orig"], fx["patch"], fx["stride"], "fundus", fx["K"], "segtran",
                                      fx["mirror_axes"], weight)


@pytest.mark.parametrize("key", ["brats_same", "brats_resized", "argmax"])
def test_unit_weights_reproduce_the_3d_reference_fixture(key):
    c = load_golden("infer_sw")["cases"][key]
    net = AffinePickNet(c["a"], c["b"], c["ch"])
    hard, soft = GO.test_single_case_gauss(net, c["image"], c["orig_patch"], c["input_patch"], c["batch_size"],
                                           c["stride_xy"], c["stride_z"], c["task"], "segtran", c["K"], (),
                                           torch.ones(c["orig_patch"]))
    assert torch.equal(soft, c["soft"]) and torch.equal(hard, c["hard"])


def test_unit_weights_reproduce_the_2d_reference_fixture():
    for key, c in load_golden("eval2d")["sw"].items():
        net = AffinePickNet(c["a"], c["b"], c["ch"])
        hard, soft = GO.test_single_batch_gauss(net, c["image"], c["orig"], c["patch"], c["stride"], "fundus", c["K"],
                                                "segtran", (), torch.ones(c["orig"]))
        assert torch.equal(soft, c["soft"]) and torch.equal(hard, c["hard"]), key


@pytest.mark.parametrize("name", TTA)
def test_unit_weights_reproduce_the_tta_fixtures(name):
    """The TTA fixtures average each variant separately, so they agree with any pooled average to rounding (1e-6, as
    the TTA oracle's own test); the pooled TTA oracle is reproduced bit for bit."""
    fx = load_golden(name)
    net = TO.AsymNet(**fx["net"])
    ones = torch.ones(fx["orig_patch"] if fx["kind"] == "tta3d" else fx["orig"])
    hard, soft = run_gauss(fx, net, fx["image"], ones)
    tta_hard, tta_soft = run_oracle(fx, net, fx["image"])
    assert torch.equal(soft, tta_soft) and torch.equal(hard, tta_hard)
    assert float((soft - fx["soft"]).abs().max()) < 1e-6
    sure = sure_mask(fx["soft"], fx["hard"], fx["kind"])
    assert torch.equal(hard[sure], fx["hard"][sure])


def _axis_f64(d, s):
    g = np.exp(-((np.arange(d, dtype=np.float64) - (d - 1) / 2) ** 2) / (2 * (s * d) ** 2))
    return torch.from_numpy(g / g.max()).float()


@pytest.mark.parametrize("size", [(112, 112, 96), (112, 112, 112), (576, 576), (288, 256), (7, 8, 1), (2, 3, 5)])
@pytest.mark.parametrize("s", [0.125, 0.25, 1.0, 0.05])
def test_tables_match_a_float64_restatement(size, s):
    from segtran_b200.inference import gaussian_window_tables
    tab = gaussian_window_tables(size, s)
    assert tab.dtype == torch.float32 and tab.shape == (sum(size),)
    for g, d in zip(torch.split(tab, list(size)), size):
        assert torch.equal(g, _axis_f64(d, s)) and torch.equal(g, GO.gaussian_axis(d, s))
        assert torch.equal(g, g.flip(0))                                    # symmetric
        assert float(g.max()) == 1.0 and float(g[(d - 1) // 2]) == 1.0     # peaks at 1 at the centre cell(s)
        assert bool((g > 0).all()) and bool((g <= 1).all())


def test_the_floor_holds_for_a_small_sigma():
    from segtran_b200.inference import gaussian_window_tables
    size, s = (24, 20, 16), 0.02
    tab = gaussian_window_tables(size, s)
    gx, gy, gz = torch.split(tab, list(size))
    raw = gx.view(-1, 1, 1) * gy.view(1, -1, 1) * gz.view(1, 1, -1)        # the kernels' product order
    w = raw.clamp_min(1e-3)
    assert float(raw.min()) < 1e-30                                         # the Gaussian itself vanishes at the corners
    assert float(w.min()) == float(torch.tensor(1e-3)) and float(w.max()) == 1.0
    assert torch.equal(w, GO.gaussian_weight(size, s))
    # a tiny sigma: the centre cells still weigh 1 (the maximum is divided out in the exponent, no 0 / 0)
    assert torch.equal(gaussian_window_tables((2,), 1e-4), torch.ones(2))
    assert torch.equal(gaussian_window_tables((3,), 1e-4), torch.tensor([0.0, 1.0, 0.0]))


BAD = [0, 0.0, -1, -0.5, float("nan"), float("inf"), -float("inf"), True, False, "0.125", (0.125,), 1j]


@pytest.mark.parametrize("s", BAD, ids=[repr(v) for v in BAD])
def test_bad_sigma_scale_raises_value_error_before_any_launch(s):
    from segtran_b200.inference import test_single_batch, test_single_case
    net = AffinePickNet([1.0, 1.0], [0.0, 0.0], [0, 0])
    with pytest.raises(ValueError, match="gaussian_sigma_scale"):
        test_single_case(net, torch.zeros(1, 8, 8, 8), (8, 8, 8), (8, 8, 8), 1, 8, 8, "other", "segtran", 2,
                         gaussian_sigma_scale=s)
    with pytest.raises(ValueError, match="gaussian_sigma_scale"):
        test_single_batch(net, torch.zeros(1, 1, 8, 8), (8, 8), (8, 8), (8, 8), "fundus", 2, "segtran",
                          mirror_axes=(1,), gaussian_sigma_scale=s)


def test_valid_sigma_scales_still_need_a_gpu():
    from segtran_b200 import _lib as L
    from segtran_b200.inference import test_single_batch, test_single_case
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    net = AffinePickNet([1.0, 1.0], [0.0, 0.0], [0, 0])
    for s in (0.125, 2, np.float64(0.5)):
        with pytest.raises(L.SxError):
            test_single_case(net, torch.zeros(1, 8, 8, 8), (8, 8, 8), (8, 8, 8), 1, 8, 8, "other", "segtran", 2,
                             gaussian_sigma_scale=s)
        with pytest.raises(L.SxError):
            test_single_batch(net, torch.zeros(1, 1, 8, 8), (8, 8), (8, 8), (8, 8), "fundus", 2, "segtran",
                              gaussian_sigma_scale=s)


def test_header_declares_the_weight_descriptor():
    import ctypes
    from segtran_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "segtran_b200.h")).read()
    assert ("typedef struct {\n  const float* wx;\n  const float* wy;\n  const float* wz;\n  int32_t nx, ny, nz, _pad;\n"
            "} sx_sw_weights;") in hdr
    assert ctypes.sizeof(_lib.sx_sw_weights) == 40
    assert (_lib.sx_sw_weights.wy.offset, _lib.sx_sw_weights.wz.offset, _lib.sx_sw_weights.nx.offset,
            _lib.sx_sw_weights.nz.offset) == (8, 16, 24, 32)
    for name in ("sx_sw_accumulate", "sx_sw2d_accumulate"):
        assert _lib._PROTOS[name][-2:] == [ctypes.POINTER(_lib.sx_sw_weights), ctypes.c_void_p]
    readme = open(os.path.join(ROOT, "README.md")).read()
    line = next(ln for ln in readme.splitlines() if "include/segtran_b200.h" in ln)
    assert "(%d entry points)" % len(_lib.EXPORTS) in line


def _refused(name, *args):
    from segtran_b200 import _lib as L
    with pytest.raises(L.SxError) as e:
        L.call(name, *args)
    return str(e.value)


def _weights(wx, nx, wy, ny, wz, nz):
    import ctypes
    from segtran_b200 import _lib as L
    return ctypes.byref(L.sx_sw_weights(wx, wy, wz, nx, ny, nz))


def test_table_size_mismatch_is_refused_before_any_launch():
    """The pointers below are never dereferenced: every call is refused on the host."""
    acc3 = (0, 4, 2, 2, 2, 0, 0, 4, 4, 4, 0, 0, 0, 0)                        # a valid 2x2x2 window in a 4x4x4 volume
    acc2 = (0, 1, 3, 2, 2, 4, 4, 0, 0, 8, 8, 0, 0, 0)                        # a valid 4x4 window in an 8x8 image
    for tables in [(8, 3, 8, 2, 8, 2), (8, 2, 8, 2, 8, 3), (8, 2, 8, 2, None, 1), (8, 2, 8, 4, 8, 2)]:
        assert "weight tables" in _refused("sx_sw_accumulate", *acc3, _weights(*tables), None)
    for tables in [(8, 4, 8, 3, None, 1), (8, 2, 8, 4, None, 1), (8, 4, 8, 4, 8, 2)]:
        assert "weight tables" in _refused("sx_sw2d_accumulate", *acc2, _weights(*tables), None)
    for tables in [(8, 2, None, 2, None, 1), (8, 0, 8, 2, None, 1), (8, 2, 8, 2, 8, 0), (None, 2, 8, 2, 8, 2)]:
        assert "missing table" in _refused("sx_sw_accumulate", *acc3, _weights(*tables), None)
        assert "missing table" in _refused("sx_sw2d_accumulate", *acc2, _weights(*tables), None)
