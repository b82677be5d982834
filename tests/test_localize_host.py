"""CPU tests of localize's host side: every request MickeyRelativePose.localize rejects raises MickeyB200Error before
anything is launched and before a seed is drawn, and mk_localize rejects its bad arguments with MK_ERR_INVALID before it
reads the handle."""
import ctypes as C

import numpy as np
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200._lib import MickeyB200Error
from mickey_b200.config import mickey_cfg
from mickey_b200.model import MickeyFeatures, MickeyRelativePose, validate_localize

MK_ERR_INVALID = -1
H, W = 42, 56                      # token grid (3, 4)


def _bank(n, grid=(3, 4), device="cpu"):
    N = grid[0] * grid[1]
    z = lambda *s: torch.zeros(*s, device=device)                    # noqa: E731
    return MickeyFeatures(z(n, 2, N), z(n, 1, N), z(n, 1, N), z(n, 128, N), grid, (grid[0] * 14, grid[1] * 14))


def _queries(p, h=H, w=W, u8=False):
    return torch.zeros(p, h, w, 3, dtype=torch.uint8) if u8 else torch.zeros(p, 3, h, w)


def _K(n):
    return torch.eye(3)[None].repeat(n, 1, 1)


def test_validate_localize_accepts_host_lists_tensors_and_both_image_formats():
    ref = _bank(2)
    assert validate_localize(ref, [0, 1, 1], _queries(3), _K(3), _K(3)) == [0, 1, 1]
    assert validate_localize(ref, torch.tensor([1], dtype=torch.int32), _queries(1, u8=True), _K(1), _K(1)) == [1]
    assert validate_localize(ref, np.array([0, 0], dtype=np.int64), _queries(2, h=H + 13, w=W + 5), _K(2), _K(2)) == [0, 0]


BAD = {
    "index_equal_to_bank_size": dict(idx=[0, 2]),
    "negative_index": dict(idx=[0, -1]),
    "float_index": dict(idx=[0.0, 1.0]),
    "float_tensor_index": dict(idx=torch.tensor([0.0, 1.0])),
    "fewer_indices_than_queries": dict(idx=[0]),
    "no_queries": dict(idx=[], queries=_queries(0)),
    "reference_grid_differs": dict(queries=_queries(2, h=H + 14)),
    "K0_of_another_pair_count": dict(K0=_K(3)),
    "K1_of_another_pair_count": dict(K1=_K(1)),
    "queries_not_images": dict(queries=torch.zeros(2, 4, H, W)),
    "uint8_queries_not_hwc": dict(queries=torch.zeros(2, 3, H, W, dtype=torch.uint8)),
    "reference_split_across_devices": dict(ref=MickeyFeatures(*_bank(2).tensors()[:3], torch.zeros(2, 128, 12, device="meta"),
                                                              (3, 4), (H, W))),
    "queries_on_another_device": dict(queries=torch.zeros(2, 3, H, W, device="meta")),
}
# a request that is well formed but whose reference is not on the model's device (the CPU here)
BAD_FOR_MODEL = {**BAD, "reference_on_another_device": dict(ref=_bank(2, device="meta"), queries=torch.zeros(2, 3, H, W, device="meta"))}


def _request(ref=None, idx=(0, 1), queries=None, K0=None, K1=None):
    ref = _bank(2) if ref is None else ref
    queries = _queries(2) if queries is None else queries
    return ref, list(idx) if isinstance(idx, tuple) else idx, queries, _K(2) if K0 is None else K0, _K(2) if K1 is None else K1


@pytest.mark.parametrize("case", sorted(BAD))
def test_validate_localize_rejects(case):
    with pytest.raises(MickeyB200Error):
        validate_localize(*_request(**BAD[case]))


@pytest.fixture(scope="module")
def model():
    return MickeyRelativePose(mickey_cfg("vits", 2, 8))               # on the CPU: it must never get as far as the engine


@pytest.mark.parametrize("case", sorted(BAD_FOR_MODEL))
def test_model_rejects_before_any_seed_is_drawn(model, case):
    rng = torch.get_rng_state()
    with pytest.raises(MickeyB200Error):
        model.localize(*_request(**BAD_FOR_MODEL[case]))
    assert torch.equal(torch.get_rng_state(), rng)


# ---- the C entry points ---------------------------------------------------------------------------------------------
def _localize_args(**kw):
    """mk_localize's 30 arguments; every pointer is a host buffer the call must not touch.  The handle is a zeroed host
    block: were the checks to fall through, the handle would read as not finalized, whose message does not name
    mk_localize."""
    buf = C.create_string_buffer(4096)
    p = C.cast(buf, C.c_void_p)
    a = dict(h=p, ref_kps=p, ref_depth=p, ref_scr=p, ref_dsc=p, n_ref=2, ref_idx=p, queries=p, K0=p, K1=p, n_pairs=3,
             H=224, W=196, seed=C.c_ulonglong(1), kps=p, depth=p, scr=None, dsc=None, scores=p, kp_scores=p, final=p,
             pitch=0, pose=p, best_set=None, inl=None, sampled=None, status=None, ws=p, ws_bytes=4096, stream=None)
    a.update(kw)
    return buf, list(a.values())


REQUIRED = ("h", "ref_kps", "ref_depth", "ref_scr", "ref_dsc", "ref_idx", "queries", "K0", "K1", "kps", "depth", "final", "pose")
C_BAD = {**{f"null_{n}": {n: None} for n in REQUIRED}, "no_pairs": {"n_pairs": 0}, "negative_pairs": {"n_pairs": -2},
         "empty_reference_bank": {"n_ref": 0}, "scores_without_kp_scores": {"kp_scores": None}}


@pytest.mark.parametrize("fn", ["mk_localize", "mk_localize_u8"])
@pytest.mark.parametrize("case", sorted(C_BAD))
def test_c_entry_rejects_before_reading_the_handle(fn, case):
    lib = _lib.load()
    keep, args = _localize_args(**C_BAD[case])
    assert getattr(lib, fn)(*args) == MK_ERR_INVALID
    assert b"mk_localize" in lib.mk_last_error()
    del keep


def test_workspace_query_rejects_a_null_handle():
    """mk_localize's workspace is mk_workspace_bytes_for(P, P); without a handle the query gives -1."""
    assert _lib.load().mk_workspace_bytes_for(None, 4, 4, 224, 196) == -1
