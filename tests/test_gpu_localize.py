"""localize: P queries against cached references, the queries alone extracted (mk_localize).  Under the same torch seed
every output must be bit-equal to model.forward on the explicit pairs (reference image, query p) and to
pose_from_features on a query bank: extraction is per image and batch-invariant, the role-0 gather rounds exactly like
the extraction's descriptor split, and the matcher and solver then run the same launches on the same operands, so any
difference is a bug, not rounding."""
import ctypes as C
import gc

import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.io import to_float_chw
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from tests.common import K_TOY

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
H, W = 224, 196
KEYS = ("kps0", "kps1", "depth_kp0", "depth_kp1", "scr0", "scr1", "dsc0", "dsc1", "depth0_map", "depth1_map", "scores",
        "kp_scores", "final_scores", "R", "t", "inliers")
LEAN_KEYS = tuple(k for k in KEYS if k not in ("scores", "kp_scores"))
_MODELS = {}


def _new_model(variant="vits", im=4, ir=16):
    cfg = mickey_cfg(variant, im, ir)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    return model.to(DEV).eval()


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """The cached models keep their engines' buffer sets, workspaces and graphs (several GB at P = 32, 720x540): drop them
    when the module ends, so that the modules after this one get the device memory back."""
    yield
    _MODELS.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _model(variant="vits", im=4, ir=16):
    key = (variant, im, ir)
    if key not in _MODELS:
        _MODELS[key] = _new_model(variant, im, ir)
    return _MODELS[key]


def _u8(n, seed, h=H, w=W):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8)


def _images(n, seed, h=H, w=W):
    return to_float_chw(_u8(n, seed, h, w)).to(DEV)


def _K(n):
    return torch.tensor(K_TOY, device=DEV)[None].repeat(n, 1, 1)


def _paired(model, im0, im1, seed=5):
    data = {"image0": im0, "image1": im1, "K_color0": _K(len(im0)), "K_color1": _K(len(im0))}
    torch.manual_seed(seed)
    model(data, return_inliers=True)
    return data


def _banked(model, ref, idx, query_bank, seed=5):
    torch.manual_seed(seed)
    return model.pose_from_features(ref, idx, query_bank, range(len(idx)), _K(len(idx)), _K(len(idx)), return_inliers=True)


def _localized(model, ref, idx, queries, seed=5, K=None):
    torch.manual_seed(seed)
    K = _K(len(idx)) if K is None else K
    return model.localize(ref, idx, queries, K, K, return_inliers=True)


def _assert_same(ref, got, keys=KEYS):
    for k in keys:
        assert torch.equal(ref[k], got[k]), k
    assert ref["kps0_shape"] == got["kps0_shape"] and ref["down_factor"] == got["down_factor"]
    assert len(ref["inliers_list"]) == len(got["inliers_list"])
    for a, b in zip(ref["inliers_list"], got["inliers_list"]):
        assert torch.equal(a, b)


def _cpu(d, keys=KEYS):
    """A call's outputs copied out (static buffers are reused by later calls)."""
    return {**{k: d[k].clone() for k in keys}, "inliers_list": [t.clone() for t in d["inliers_list"]],
            "kps0_shape": d["kps0_shape"], "down_factor": d["down_factor"]}


# ---- equal to forward on the explicit pairs --------------------------------------------------------------------------
@pytest.mark.parametrize("geo", [(720, 540), (658, 686)])
@pytest.mark.parametrize("u8", [False, True])
@pytest.mark.parametrize("P", [1, 3, 32])
def test_equals_forward_on_explicit_pairs(P, u8, geo):
    model = _model()
    h, w = geo
    ref_u8, q_u8 = _u8(1, 100 + P, h, w), _u8(P, 200 + P, h, w)
    if u8:
        ref_img, queries = ref_u8.to(DEV), q_u8.to(DEV)
    else:
        ref_img, queries = to_float_chw(ref_u8).to(DEV), to_float_chw(q_u8).to(DEV)
    paired = _paired(model, ref_img.expand(P, *ref_img.shape[1:]).contiguous(), queries)
    ref = model.extract_features(ref_img)
    assert ref.grid == (h // 14, w // 14)
    _assert_same(paired, _localized(model, ref, [0] * P, queries))


# ---- equal to feature banks --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lean", [False, True])
@pytest.mark.parametrize("variant", ["vits", "vitb"])
def test_equals_pose_from_features_two_references_interleaved(variant, lean):
    model = _model(variant)
    refs, queries = _images(2, 11), _images(6, 12)
    idx = [0, 1, 0, 1, 1, 0]
    ref = model.extract_features(refs)
    query_bank = model.extract_features(queries)
    model.lean_outputs = lean
    try:
        banked = _banked(model, ref, idx, query_bank)
        got = _localized(model, ref, idx, queries)
    finally:
        model.lean_outputs = False
    keys = LEAN_KEYS if lean else KEYS
    _assert_same(banked, got, keys)
    assert ("scores" in got) == (not lean) and set(got) == set(banked)
    assert torch.equal(got["scr1"], query_bank.scr) and torch.equal(got["dsc1"], query_bank.dsc)


def _raw_localize(eng, ref, idx_dev, queries, seed, scr_dsc=True, lean=False):
    """One eager mk_localize call on fresh outputs, its own workspace: (outputs, return code)."""
    P, N = queries.shape[0], ref.kps.shape[-1]
    H_, W_ = queries.shape[-2], queries.shape[-1]
    eng._use_geometry(H_, W_)
    ws = _lib.workspace(eng.lib.mk_workspace_bytes_for(eng.h, P, P, H_, W_), DEV, "mk_workspace_bytes_for")
    out = eng._outputs(2 * P, P, N, lean, scr_dsc=False)
    if scr_dsc:
        out["scr"], out["dsc"] = torch.empty(P, 1, N, device=DEV), torch.empty(P, 128, N, device=DEV)
    else:
        out["scr"], out["dsc"] = None, None
    out = {k: out[k] for k in ("kps", "depth", "scr", "dsc", "scores", "kp_scores", "final_scores", "pose", "best_set",
                                "inlier_mask", "sampled_idx", "status")}
    p, K = _lib.ptr, _K(P)
    rc = eng.lib.mk_localize(eng.h, *(p(t) for t in ref.tensors()), len(ref), p(idx_dev), p(queries.contiguous()), p(K), p(K), P,
                             H_, W_, C.c_ulonglong(seed), *eng._output_args(out), p(ws), ws.numel(), _lib.stream())
    torch.cuda.synchronize()
    return out, rc


def test_query_features_are_optional_in_the_c_call():
    model = _model()
    eng = model._engine()
    ref, queries = model.extract_features(_images(2, 31)), _images(3, 32)
    idx = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
    full, rc0 = _raw_localize(eng, ref, idx, queries, 77)
    bare, rc1 = _raw_localize(eng, ref, idx, queries, 77, scr_dsc=False)
    assert rc0 == 0 and rc1 == 0
    for k in ("kps", "depth", "scores", "kp_scores", "final_scores", "pose", "best_set", "inlier_mask", "sampled_idx", "status"):
        assert torch.equal(full[k], bare[k]), k
    query_bank = model.extract_features(queries)
    assert torch.equal(full["scr"], query_bank.scr) and torch.equal(full["dsc"], query_bank.dsc)


def test_out_of_range_index_in_the_c_call_gives_the_zero_pose():
    model = _model()
    eng = model._engine()
    ref, queries = model.extract_features(_images(2, 41)), _images(3, 42)
    ok, _ = _raw_localize(eng, ref, torch.tensor([0, 1, 1], dtype=torch.int32, device=DEV), queries, 9)
    assert int(ok["status"].item()) & 8 == 0
    for bad in ([0, 2, 1], [0, 1, -1]):
        out, rc = _raw_localize(eng, ref, torch.tensor(bad, dtype=torch.int32, device=DEV), queries, 9)
        assert rc == 0
        assert int(out["status"].item()) & 8
        assert torch.equal(out["pose"], torch.zeros_like(out["pose"]))


def test_workspace_holds_p_role_one_images():
    eng = _model()._engine()
    lib, h = eng.lib, eng.h
    for P in (1, 3, 32):
        loc, fwd = lib.mk_workspace_bytes_for(h, P, P, 720, 540), lib.mk_workspace_bytes(h, P, 720, 540)
        assert lib.mk_workspace_bytes_for(h, 0, P, 720, 540) < loc < fwd


# ---- graphs, pipelining and host frames ----------------------------------------------------------------------------------
SEEDS = (3, 4, 5, 6, 7)


def _sequence(model, ref, idx, queries_of, keys=KEYS, sync=True):
    outs = []
    for i, s in enumerate(SEEDS):
        outs.append(_cpu(_localized(model, ref, idx, queries_of(i), seed=s), keys))
        if sync:
            torch.cuda.synchronize()
    return outs


def test_graph_replays_equal_eager_calls():
    model = _model()
    ref = model.extract_features(_images(2, 51))
    qs = [_images(4, 60 + i) for i in range(len(SEEDS))]
    idx = [1, 0, 0, 1]
    model.use_graph = False
    try:
        eager = _sequence(model, ref, idx, lambda i: qs[i])
    finally:
        model.use_graph = True
    eng = model._engine()
    r0 = getattr(eng, "graph_replays", 0)
    graphed = _sequence(model, ref, idx, lambda i: qs[i])
    assert getattr(eng, "graph_replays", 0) - r0 >= 2
    for a, b in zip(eager, graphed):
        _assert_same(a, b)


@pytest.mark.parametrize("depth", [2, 3])
@pytest.mark.parametrize("mode", ["default", "assume_inputs_ready", "static_outputs"])
def test_pipelined_host_uint8_frames_equal_eager(depth, mode):
    model = _new_model()
    ref_u8 = _u8(1, 71)
    ref = model.extract_features(ref_u8.to(DEV))
    qs = [_u8(4, 80 + i).pin_memory() for i in range(len(SEEDS))]
    idx = [0, 0, 0, 0]
    model.use_graph = False
    eager = _sequence(model, ref, idx, lambda i: qs[i].to(DEV))
    model.use_graph = True
    model.pipeline_depth = depth
    if mode != "default":
        setattr(model, mode, True)
    K = _K(4).cpu().pin_memory()
    got = []
    for i, s in enumerate(SEEDS):
        torch.manual_seed(s)
        d = model.localize(ref, idx, qs[i], K, K, return_inliers=True)
        got.append(_cpu(d))
        torch.cuda.synchronize()                # static outputs: read before the set is reused
    for a, b in zip(eager, got):
        _assert_same(a, b)


# ---- engine state: the reference slot, and other calls on the same engine ---------------------------------------------------
def test_in_place_edit_of_the_reference_between_replays():
    model = _new_model()
    ref = model.extract_features(_images(1, 91))
    queries = _images(3, 92)
    query_bank = model.extract_features(queries)
    for s in SEEDS[:3]:                                       # eager, capture, replay
        _localized(model, ref, [0, 0, 0], queries, seed=s)
    ref.dsc.mul_(0.5)
    ref.scr.add_(1e-3)
    got = _cpu(_localized(model, ref, [0, 0, 0], queries, seed=SEEDS[3]))
    _assert_same(_banked(model, ref, [0, 0, 0], query_bank, seed=SEEDS[3]), got)


def test_switching_references_and_back_reuses_nothing_stale():
    model = _new_model()
    ref_a, ref_b = model.extract_features(_images(1, 101)), model.extract_features(_images(1, 102))
    queries = _images(2, 103)
    query_bank = model.extract_features(queries)
    order = [ref_a, ref_a, ref_a, ref_b, ref_b, ref_a, ref_b]
    for i, r in enumerate(order):
        got = _cpu(_localized(model, r, [0, 0], queries, seed=10 + i))
        _assert_same(_banked(model, r, [0, 0], query_bank, seed=10 + i), got)
    # a new bank at a freed bank's address holds other features
    del ref_a, order, r
    ref_c = model.extract_features(_images(1, 104))
    got = _cpu(_localized(model, ref_c, [0, 0], queries, seed=30))
    _assert_same(_banked(model, ref_c, [0, 0], query_bank, seed=30), got)


def test_interleaving_with_forward_and_pose_from_features():
    images = _images(4, 111)
    ref_img, queries = images[:1], images[1:]

    def run(model, which):
        ref = model.extract_features(ref_img)
        query_bank = model.extract_features(queries)
        out = {}
        for i, s in enumerate(SEEDS):
            for w in which:
                if w == "L":
                    out[(w, i)] = _cpu(_localized(model, ref, [0, 0, 0], queries, seed=s))
                elif w == "F":
                    out[(w, i)] = _cpu(_paired(model, ref_img.expand(3, -1, -1, -1).contiguous(), queries, seed=s))
                else:
                    out[(w, i)] = _cpu(_banked(model, ref, [0, 0, 0], query_bank, seed=s))
        return out

    mixed = run(_new_model(), "LFP")
    alone = {}
    for w in "LFP":
        alone.update(run(_new_model(), w))
    assert set(mixed) == set(alone)
    for k in mixed:
        _assert_same(alone[k], mixed[k])
    for i in range(len(SEEDS)):
        _assert_same(mixed[("F", i)], mixed[("L", i)])


def test_full_size_c3_one_reference_thirty_two_queries():
    """BASELINE config 3's model: ViT-B, 720x540, 1024 hypotheses; 32 queries against one reference, graph-replayed."""
    model = _model("vitb", 16, 64)
    ref_img, queries = _images(1, 121, 720, 540), _images(32, 122, 720, 540)
    ref = model.extract_features(ref_img)
    query_bank = model.extract_features(queries)
    for s in SEEDS[:3]:
        got = _cpu(_localized(model, ref, [0] * 32, queries, seed=s))
        _assert_same(_banked(model, ref, [0] * 32, query_bank, seed=s), got)
    assert tuple(got["final_scores"].shape) == (32, 1938, 1938)
