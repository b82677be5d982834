"""The rules of the library boundary that mickey_b200/_lib.py owns for every caller: which [B, N, N] layouts go to the
library as they are and at what row pitch, workspace allocation, and the struct layouts the ctypes binding shares with
the library.  No GPU needed."""
import ctypes

import pytest
import torch

from mickey_b200 import _lib

B, N, P = 3, 10, 16


def _kept(t, pitch):
    out, p = _lib.pitched(t)
    assert out is t and p == pitch


def _copied(t):
    out, p = _lib.pitched(t)
    assert out is not t and out.is_contiguous() and torch.equal(out, t) and p == N


def test_pitched_reads_contiguous_tensors_and_padded_views_in_place():
    _kept(torch.rand(B, N, N), N)
    _kept(torch.rand(B, N, P)[:, :, :N], P)                          # the engine's [B, N, pitch][:, :, :N] outputs
    _kept(torch.rand(4 * N * P).as_strided((1, N, N), (7, P, 1)), P)  # one matrix: stride(0) is never used


def test_pitched_copies_layouts_the_library_cannot_read():
    _copied(torch.rand(B, N, N).transpose(1, 2))                      # columns contiguous
    t = torch.rand(N).expand(B, N, N)                                 # every row one vector: pitch 0 would read past it
    assert t.stride() == (0, 0, 1)
    _copied(t)


def test_workspace_raises_on_a_rejected_geometry_and_never_hands_out_null():
    lib = _lib.load()
    nbytes = lib.mk_resblock_ws_bytes(0, 1, 1, 32, 32)                # B = 0: the library answers -1
    assert nbytes == -1
    with pytest.raises(_lib.MickeyB200Error, match="mk_resblock_ws_bytes returned -1"):
        _lib.workspace(nbytes, "cpu", "mk_resblock_ws_bytes")
    assert _lib.workspace(0, "cpu", "x").numel() == 1
    ws = _lib.workspace(lib.mk_resblock_ws_bytes(1, 4, 4, 32, 32), "cpu", "mk_resblock_ws_bytes")
    assert ws.dtype == torch.uint8 and ws.numel() == lib.mk_resblock_ws_bytes(1, 4, 4, 32, 32)


@pytest.mark.parametrize("name,struct", [
    ("mk_config", _lib.MkConfig), ("mk_gemm_args", _lib.MkGemmArgs), ("mk_htr_layer", _lib.MkHtrLayer),
    ("mk_htr_layer_grads", _lib.MkHtrLayerGrads), ("mk_resblock_params", _lib.MkResblockParams),
    ("mk_resblock_grads", _lib.MkResblockGrads)])
def test_every_ctypes_struct_matches_the_library(name, struct):
    assert _lib.load().mk_sizeof(name.encode()) == ctypes.sizeof(struct)


def test_sizeof_an_unknown_struct_is_minus_one():
    assert _lib.load().mk_sizeof(b"nope") == -1


@pytest.mark.parametrize("epi", [8, 9])
def test_gemm_rejects_an_unknown_epilogue_before_any_launch(epi):
    """The epilogue list ends at 7 (DUAL): a well-formed GEMM with any other epi is refused on the host."""
    lib = _lib.load()
    g = _lib.MkGemmArgs()
    g.epi, g.M, g.N, g.k_chunks, g.chunks_per_tap, g.num_taps, g.groups = epi, 128, 128, 1, 1, 1, 1
    assert lib.mk_op_gemm(ctypes.byref(g), None) == -1
    assert lib.mk_last_error().decode() == f"unknown epilogue {epi}"
