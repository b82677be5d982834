"""Feature banks: extract_features once per image, pose_from_features for any pairs among them.  Under the same torch
seed every output must be bit-equal to model.forward on the explicit pairs: features do not depend on the batch
(test_batch_invariance_and_c3_shapes), and with the same pair count, seed and operands the matcher and solver launches
are the same, so any difference is a bug, not rounding."""
import pytest
import torch

from mickey_b200._lib import MickeyB200Error
from mickey_b200.config import mickey_cfg
from mickey_b200.io import to_float_chw
from mickey_b200.model import MickeyFeatures, MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from tests.common import K_TOY

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
H, W = 224, 196
KEYS = ("kps0", "kps1", "depth_kp0", "depth_kp1", "scr0", "scr1", "dsc0", "dsc1", "depth0_map", "depth1_map", "scores",
        "kp_scores", "final_scores", "R", "t", "inliers")
_MODELS = {}


def _model(variant="vits", im=4, ir=16):
    key = (variant, im, ir)
    if key not in _MODELS:
        cfg = mickey_cfg(variant, im, ir)
        model = MickeyRelativePose(cfg)
        model.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
        _MODELS[key] = model.to(DEV).eval()
    return _MODELS[key]


def _images(n, seed, h=H, w=W):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, h, w, generator=g).to(DEV)


def _K(n):
    return torch.tensor(K_TOY, device=DEV)[None].repeat(n, 1, 1)


def _paired(model, im0, im1, seed=5):
    data = {"image0": im0, "image1": im1, "K_color0": _K(len(im0)), "K_color1": _K(len(im0))}
    torch.manual_seed(seed)
    model(data, return_inliers=True)
    return data


def _banked(model, f0, i0, f1, i1, seed=5):
    torch.manual_seed(seed)
    return model.pose_from_features(f0, i0, f1, i1, _K(len(i0)), _K(len(i0)), return_inliers=True)


def _assert_same(ref, got, keys=KEYS):
    for k in keys:
        assert torch.equal(ref[k], got[k]), k
    assert ref["kps0_shape"] == got["kps0_shape"] and ref["down_factor"] == got["down_factor"]
    assert len(ref["inliers_list"]) == len(got["inliers_list"])
    for a, b in zip(ref["inliers_list"], got["inliers_list"]):
        assert torch.equal(a, b)


# pairs as (reference of each pair, query of each pair) over refs r0, r1 and queries q0..q3
CASES = {"one_reference": [0, 0, 0, 0], "two_references": [0, 0, 1, 1]}


def _case(name):
    refs, queries = _images(2, 11), _images(4, 12)
    ref_of = CASES[name]
    return refs, queries, ref_of


@pytest.mark.parametrize("name", sorted(CASES))
def test_shared_reference_equals_paired_path(name):
    model = _model()
    refs, queries, ref_of = _case(name)
    ref = _paired(model, refs[ref_of], queries)
    feats = model.extract_features(torch.cat([refs, queries]))            # the 6 distinct images, once each
    assert len(feats) == 6 and feats.grid == (H // 14, W // 14)
    got = _banked(model, feats, ref_of, feats, [2, 3, 4, 5])
    _assert_same(ref, got)


def test_roles_swap_within_one_bank():
    model = _model()
    ims = _images(3, 21)
    pairs = [(0, 1), (1, 0), (2, 2), (1, 2)]
    i0, i1 = [a for a, _ in pairs], [b for _, b in pairs]
    ref = _paired(model, ims[i0], ims[i1])
    feats = model.extract_features(ims)                                    # odd image count
    _assert_same(ref, _banked(model, feats, i0, feats, torch.tensor(i1)))


@pytest.mark.parametrize("name", sorted(CASES))
def test_cached_reference_bank_across_calls(name):
    model = _model()
    refs, queries, ref_of = _case(name)
    ref = _paired(model, refs[ref_of], queries)
    ref_bank = model.extract_features(refs)                                # 2 images in one call ...
    _paired(model, queries, queries)                                       # ... other work on the engine in between ...
    query_bank = model.extract_features(queries)                           # ... 4 in a later one: another carving
    _assert_same(ref, _banked(model, ref_bank, ref_of, query_bank, range(4)))


def test_uint8_input_is_bit_equal_to_float():
    model = _model()
    g = torch.Generator().manual_seed(31)
    u8 = torch.randint(0, 256, (3, H, W, 3), generator=g, dtype=torch.uint8)
    ims = to_float_chw(u8)                          # the reference's float tensor, normalised on the host
    a, b = model.extract_features(ims.to(DEV)), model.extract_features(u8.to(DEV))
    for x, y in zip(a.tensors(), b.tensors()):
        assert torch.equal(x, y)
    assert a.grid == b.grid and a.image_size == b.image_size == (H, W)


def test_lean_mode_drops_scores_only():
    model = _model()
    refs, queries, ref_of = _case("two_references")
    feats = model.extract_features(torch.cat([refs, queries]))
    full = _banked(model, feats, ref_of, feats, [2, 3, 4, 5])
    model.lean_outputs = True
    try:
        lean = _banked(model, feats, ref_of, feats, [2, 3, 4, 5])
    finally:
        model.lean_outputs = False
    assert "scores" not in lean and "kp_scores" not in lean
    _assert_same(full, lean, [k for k in KEYS if k not in ("scores", "kp_scores")])


def test_rejected_requests_raise_before_any_launch():
    model = _model()
    feats = model.extract_features(_images(3, 41))
    other = model.extract_features(_images(2, 42, h=210, w=196))         # another token grid
    eng = model._engine()
    torch.cuda.synchronize()
    launches, rng = eng.launch_count, torch.get_rng_state()
    bad = [
        (feats, [0, 3], feats, [1, 2]),            # index == bank size
        (feats, [0, -1], feats, [1, 2]),           # negative index
        (feats, [0, 1], feats, [1]),               # unequal lengths
        (feats, [], feats, []),                    # no pair
        (feats, [0.0], feats, [1]),                # not integers
        (feats, [0], other, [1]),                  # banks of different geometry
    ]
    for f0, i0, f1, i1 in bad:
        with pytest.raises(MickeyB200Error):
            model.pose_from_features(f0, i0, f1, i1, _K(max(len(i0), 1)), _K(max(len(i0), 1)))
    cpu = MickeyFeatures(*(t.cpu() for t in feats.tensors()), feats.grid, feats.image_size)
    with pytest.raises(MickeyB200Error):
        model.pose_from_features(cpu, [0], feats, [1], _K(1), _K(1))         # banks on two devices
    with pytest.raises(MickeyB200Error):
        model.pose_from_features(feats, [0, 1], feats, [1, 2], _K(1), _K(1))  # K of another pair count
    assert eng.launch_count == launches
    assert torch.equal(torch.get_rng_state(), rng)                      # no seed was drawn


def test_workspace_queries():
    eng = _model()._engine()
    lib, h = eng.lib, eng.h
    for P in (1, 4, 32):
        assert lib.mk_workspace_bytes(h, P, 720, 540) == lib.mk_workspace_bytes_for(h, 2 * P, P, 720, 540)
        assert 0 < lib.mk_workspace_bytes_for(h, 0, P, 720, 540) < lib.mk_workspace_bytes(h, P, 720, 540)
    assert lib.mk_workspace_bytes_for(h, 3, 0, 720, 540) < lib.mk_workspace_bytes_for(h, 4, 0, 720, 540)


def test_full_size_c3_one_reference_eight_queries():
    """BASELINE config 3's model at full size: ViT-B, 720x540, 1024 hypotheses; 8 queries against one reference."""
    model = _model("vitb", 16, 64)
    ref_img, queries = _images(1, 51, 720, 540), _images(8, 52, 720, 540)
    ref = _paired(model, ref_img.expand(8, -1, -1, -1).contiguous(), queries)
    ref_bank, query_bank = model.extract_features(ref_img), model.extract_features(queries)
    got = _banked(model, ref_bank, [0] * 8, query_bank, range(8))
    assert tuple(got["final_scores"].shape) == (8, 1938, 1938)
    _assert_same(ref, got)
