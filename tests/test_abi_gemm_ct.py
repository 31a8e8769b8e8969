"""CPU-side check of sx_gemm's transposed-output block (its `tout` argument): the ctypes mirror has the C layout of
include/segtran_b200.h, and sx_gemm_args keeps its own."""


def test_gemm_tout_layout_matches_header():
    import ctypes as C
    from segtran_b200 import _lib
    assert C.sizeof(_lib.sx_gemm_tout) == 32
    assert _lib.sx_gemm_tout.ldct.offset == 8 and _lib.sx_gemm_tout.ct_stride_z1.offset == 24
    assert C.sizeof(_lib.sx_gemm_args) == 256
    assert _lib._PROTOS["sx_gemm"] == [C.POINTER(_lib.sx_gemm_args), C.POINTER(_lib.sx_gemm_tout), C.c_void_p]
