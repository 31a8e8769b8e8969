"""CPU checks of the 3-D batch preparation (segtran_b200/datasets3d.py): the stock-PyTorch restatement
(oracle/prep3d_oracle.py) against the fixtures built from the reference's own brats_map_label and RandomResizedCrop
(oracle/gen_prep3d_golden.py), the C-ABI declarations of the new entry points, and the argument errors, which are raised
before anything needs a device."""
import ctypes as C
import glob
import os
import re

import pytest
import torch

from oracle import prep3d_oracle as PO
from tests.helpers import GOLDEN, load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CROPS = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(GOLDEN, "prep3d_crop_*.pt")))
NEW_ENTRY_POINTS = ["sx_brats_map_label", "sx_draw_resized_crop", "sx_resized_crop"]


def test_fixture_set_covers_the_cases():
    assert CROPS == ["prep3d_crop_aniso", "prep3d_crop_down", "prep3d_crop_odd", "prep3d_crop_up"]
    batches = {load_golden(n)["volume"].shape[0] for n in CROPS}
    assert {1, 3} <= batches


@pytest.mark.parametrize("key", ["batched", "unbatched"])
def test_oracle_label_maps_match_the_reference(key):
    c = load_golden("prep3d_labels")["cases"][key]
    assert set(c["labels"].unique().tolist()) == {0, 1, 2, 3, 4, 255}
    for binarize, ref in ((False, c["map4"]), (True, c["map2"])):
        got = PO.brats_map_label(c["labels"], binarize, dtype=torch.float64)
        assert torch.equal(got.float(), ref)


@pytest.mark.parametrize("name", CROPS)
def test_oracle_resized_crop_matches_the_reference(name):
    fx = load_golden(name)
    v3, m3 = PO.resized_crop(fx["volume"].double(), fx["mask"].double(), fx["out_size"], fx["draws"],
                             resize=PO.trilinear_f32_taps)
    assert v3.shape == fx["volume3"].shape and m3.shape == fx["mask3"].shape
    assert float((v3 - fx["volume3"].double()).abs().max()) <= 1e-6
    assert float((m3 - fx["mask3"].double()).abs().max()) <= 1e-6
    # the float32 F.interpolate formulation is the reference's own computation on the CPU
    v3, m3 = PO.resized_crop(fx["volume"], fx["mask"].permute(1, 0, 2, 3, 4).contiguous().permute(1, 0, 2, 3, 4),
                             fx["out_size"], fx["draws"])
    assert torch.equal(v3, fx["volume3"]) and torch.equal(m3, fx["mask3"])


def test_fixture_geometries():
    """scale > 1 everywhere, scale < 1 everywhere (the padding branch), and three scales with one axis padded."""
    geo = {}
    for name in CROPS:
        fx = load_golden(name)
        resized, pads, _ = PO.crop_geometry(fx["volume"].shape[2:], fx["out_size"], fx["draws"])
        geo[name] = "".join("p" if p != (0, 0) else "c" for p in pads)
    assert geo["prep3d_crop_up"] == "ccc" and geo["prep3d_crop_down"] == "ppp" and geo["prep3d_crop_aniso"] == "pcc"
    assert not load_golden("prep3d_crop_aniso")["isotropic"]


def _header_decls():
    hdr = open(os.path.join(ROOT, "include", "segtran_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    return hdr, dict((m.group(1), m.group(2)) for m in re.finditer(r"\bint\s+(sx_\w+)\s*\(([^;{]*?)\)\s*;", hdr, flags=re.S))


def test_header_and_ctypes_prototypes_agree():
    from segtran_b200 import _lib
    hdr, decls = _header_decls()
    for name in NEW_ENTRY_POINTS:
        assert name in decls and name in _lib._PROTOS and name in _lib.EXPORTS, name
        params = [p.strip() for p in decls[name].split(",")]
        proto = _lib._PROTOS[name]
        assert len(params) == len(proto), name
        for p, t in zip(params, proto):
            if p.startswith("int32_t"):
                assert t is C.c_int32, (name, p)
            elif p.startswith("int64_t"):
                assert t is C.c_int64, (name, p)
            elif p.startswith("uint64_t "):
                assert t is C.c_uint64, (name, p)
            elif p.startswith("float "):
                assert t is C.c_float, (name, p)
            else:
                assert "*" in p, (name, p)
    # sx_crop_operand: pointer, 5 int64 strides, pointer, two int32
    assert C.sizeof(_lib.sx_crop_operand) == 64
    assert _lib.sx_crop_operand.stride.offset == 8 and _lib.sx_crop_operand.y.offset == 48
    assert _lib.sx_crop_operand.C.offset == 56
    for v, n in enumerate(("U8", "I16", "I32", "I64", "F32")):
        assert re.search(r"SX_LABEL_%s\s*=\s*%d\b" % (n, v), hdr)
        assert getattr(_lib, "SX_LABEL_" + n) == v


def test_argument_errors_without_a_device():
    from segtran_b200 import _lib
    from segtran_b200.datasets3d import RandomResizedCrop, brats_map_label, draw_resized_crop
    v = torch.zeros(2, 1, 8, 8, 8)
    m = torch.zeros(2, 4, 8, 8, 8)
    with pytest.raises(ValueError):                         # 1 + min_crop <= 0
        RandomResizedCrop(v, m, (8, 8, 8), (-1.0, 0.1))
    with pytest.raises(ValueError):
        draw_resized_crop((8, 8, 8), (8, 8, 8), (-1.5, 0.1))
    with pytest.raises(ValueError):                         # batch mismatch
        RandomResizedCrop(v, m[:1], (8, 8, 8), (-0.1, 0.1))
    with pytest.raises(ValueError):                         # spatial mismatch
        RandomResizedCrop(v, m[..., :7], (8, 8, 8), (-0.1, 0.1))
    with pytest.raises(ValueError):                         # not 5-D
        RandomResizedCrop(v[0], m[0], (8, 8, 8), (-0.1, 0.1))
    with pytest.raises(ValueError):                         # a record of the wrong length
        RandomResizedCrop(v, m, (8, 8, 8), (-0.1, 0.1), draws=[1.0, 1.0, 1.0, 0.0, 0.0])
    with pytest.raises(ValueError):
        brats_map_label(torch.zeros(2, 2, 8, 8, 8, dtype=torch.uint8), False)
    with pytest.raises(ValueError):
        brats_map_label(torch.zeros(8, 8, 8, dtype=torch.bool), False)
    if torch.cuda.is_available():
        return
    with pytest.raises(_lib.SxError):                       # valid arguments on the CPU: no fallback
        RandomResizedCrop(v, m, (8, 8, 8), (-0.1, 0.1), draws=[1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
    with pytest.raises(_lib.SxError):
        brats_map_label(torch.zeros(2, 8, 8, 8, dtype=torch.uint8), True)
