"""segtran_b200 — H100-native (sm_90a) implementation of Segtran's Squeeze-and-Expansion hot path.

    segtran_b200.networks.segtran_shared   drop-in SegtranFusionEncoder & friends (reference module surface)
    segtran_b200.networks.segtran3d / 2d   drop-in Segtran3d / Segtran2d shells
    segtran_b200.ops                       autograd operators backed by the CUDA kernels
    segtran_b200._lib                      ctypes binding of libsegtran_b200.so (include/segtran_b200.h)
"""
__version__ = "0.1.0"
