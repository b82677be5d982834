"""Helpers for the GPU tests: thin wrappers over the operator-level C-ABI entry points."""
import ctypes as C

import torch

from mickey_b200 import _lib

EPI = dict(STORE_H=0, RESID_F=1, PATCH=2, CONV=3, STORE_F=4, LN=5, LSE=6, DUAL=7)
IMPL = dict(default=0, tc=1, simt=2)


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def gemm(epi, a, b, M, N, K=None, impl="tc", taps=None, chunks_per_tap=None, **kw):
    """a [rows, cols] fp16, b [rows, cols] fp16 (both row-major, K contiguous)."""
    lib = _lib.load()
    g = _lib.MkGemmArgs()
    g.epi, g.impl = EPI[epi], IMPL[impl]
    g.a, g.a_rows, g.a_cols, g.a_ld = a.data_ptr(), a.shape[0], a.shape[1], a.stride(0)
    g.b, g.b_rows, g.b_cols, g.b_ld = b.data_ptr(), b.shape[0], b.shape[1], b.stride(0)
    g.M, g.N = M, N
    if taps is None:
        g.num_taps, g.k_chunks = 1, K // 64
        g.chunks_per_tap = g.k_chunks
    else:
        g.num_taps, g.chunks_per_tap = len(taps), chunks_per_tap
        g.k_chunks = len(taps) * chunks_per_tap
        for i, t in enumerate(taps):
            g.tap_shift[i] = t
    g.groups = kw.pop("groups", 1)
    keep = []
    for k, v in kw.items():
        if torch.is_tensor(v):
            keep.append(v)
            v = v.data_ptr()
        setattr(g, k, v)
    _lib.check(lib.mk_op_gemm(C.byref(g), stream()), f"mk_op_gemm({epi},{impl})")
    return keep
