"""CPU-side checks of the C-ABI boundary: the library loads, exports every symbol include/segtran_b200.h declares,
and the product path refuses to run without a GPU (no silent CPU fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "segtran_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sx_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from segtran_b200 import _lib
    l = _lib.lib()
    names = _declared()
    assert len(names) >= 25
    for n in names:
        assert hasattr(l, n), "missing export %s" % n
    # the ctypes prototype table and the header agree
    assert sorted(_lib.EXPORTS) == names
    assert l.sx_version() == 1


def test_gemm_args_struct_layout_matches_header():
    import ctypes as C
    from segtran_b200 import _lib
    assert C.sizeof(_lib.sx_operand) == 40
    assert C.sizeof(_lib.sx_gemm_args) == 264 and _lib.sx_gemm_args.part.offset == 248
    assert _lib.sx_gemm_args.A.offset == 24 and _lib.sx_gemm_args.C.offset == 104


def test_no_cpu_fallback():
    from segtran_b200 import _lib, ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.SxError):
        ops.gemm_nt(torch.zeros(8, 8), torch.zeros(8, 8))
    import segtran_b200.networks.segtran_shared as S
    from tests.helpers import encoder_config
    enc = S.SegtranFusionEncoder(encoder_config(S.SegtranConfig, dims=[16, 16], num_attractors=4), "Fusion")
    with pytest.raises(Exception):
        enc(torch.zeros(1, 8, 16), torch.ones(1, 8, 3), torch.ones(1, 8, 1), torch.Size((2, 2, 2)))


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "segtran_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                assert "oracle" not in re.sub(r'""".*?"""', "", txt, flags=re.S), os.path.join(dp, f)


def test_ctypes_prototypes_match_the_header_arity():
    """Every `int sx_*(...)` declaration of include/segtran_b200.h has a ctypes prototype with the same number of
    parameters (a stale binding would shift every later argument)."""
    import os
    import re
    from segtran_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "segtran_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    decls = dict((m.group(1), m.group(2)) for m in re.finditer(r"\bint\s+(sx_\w+)\s*\(([^;{]*?)\)\s*;", hdr, flags=re.S))
    assert set(_lib._PROTOS) <= set(decls), sorted(set(_lib._PROTOS) - set(decls))
    for name, proto in _lib._PROTOS.items():
        params = decls[name].strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert n == len(proto), "%s: header declares %d parameters, ctypes prototype has %d" % (name, n, len(proto))
