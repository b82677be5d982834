"""CPU side of MicKey's correspondences (featureMatcher.get_matches_list): the oracle against the live reference's
recorded output, and the host checks of the CUDA entry points, which reject bad arguments before anything is launched."""
import math
import os

import numpy as np
import pytest
import torch

from mickey_b200.config import mickey_cfg
from mickey_b200.matches import mutual_matches
from mickey_b200.model import MickeyRelativePose, featureMatcher
from mickey_b200.weights import synthetic_state_dict
from oracle import matches_oracle
from oracle import mickey_oracle as mo
from tests.common import GOLDEN_CASES, GOLDEN_DIR, float64_eval, synthetic_pair, to_float64

FIXTURE = os.path.join(GOLDEN_DIR, "reference_matches_720x540.npz")


def assert_same_list(ours, ref, ref_row_scores):
    """ours / ref int [M, 2]; ref_row_scores: score of row i.  Tie-free positions compare exactly; a block of equal scores
    (whose order the reference's unstable sort leaves open) compares as a set."""
    ours, ref = np.asarray(ours), np.asarray(ref)
    assert ours.shape == ref.shape
    if not len(ref):
        return
    sc = ref_row_scores[ref[:, 0]]
    starts = np.flatnonzero(np.r_[True, sc[1:] != sc[:-1], True])
    for a, b in zip(starts[:-1], starts[1:]):
        if b - a == 1:
            assert tuple(ours[a]) == tuple(ref[a]), (a, ours[a], ref[a])
        else:
            assert set(map(tuple, ours[a:b])) == set(map(tuple, ref[a:b])), (a, b)


@pytest.fixture(scope="module")
def oracle_matrices():
    """The oracle's final_scores / scores of the 720x540 ViT-S and ViT-B golden cases, in float64 like the fixture."""
    out = {}
    for name in ("vits_720x540", "vitb_720x540"):
        spec = GOLDEN_CASES[name]
        cfg = mickey_cfg(spec["variant"], spec["it_matches"], spec["it_ransac"], float16=False)
        sd = to_float64(synthetic_state_dict(cfg, seed=spec["weight_seed"]))
        data = to_float64(synthetic_pair(spec["batch"], spec["height"], spec["width"], seed=spec["data_seed"]))
        with torch.no_grad(), float64_eval():
            out[name] = mo.compute_correspondences(sd, data, cfg)
    return out


@pytest.mark.parametrize("name", ["vits_720x540", "vitb_720x540"])
@pytest.mark.parametrize("mat", ["final_scores", "scores"])
def test_oracle_matches_live_reference(oracle_matrices, name, mat):
    ref = np.load(FIXTURE)
    s = oracle_matrices[name][mat]
    for b in range(s.shape[0]):
        row_scores = ref[f"{name}/{mat}/{b}/scores"]
        # the oracle's row maxima agree with the reference's to float64 rounding: the same matrix, up to ~1e-15
        assert np.allclose(s[b, :-1, :-1].max(1).values.numpy(), row_scores, rtol=1e-9, atol=1e-300)
        confs = ref[f"{name}/{mat}/{b}/min_conf"]
        for k, c in enumerate(confs):
            m, v = matches_oracle.matches_list(s[b:b + 1], float(c))
            assert_same_list(m.numpy(), ref[f"{name}/{mat}/{b}/{k}/matches"], row_scores)
            assert torch.equal(v, s[b, m[:, 0], m[:, 1]])
            assert bool((v[1:] <= v[:-1]).all())
        # min_conf = 0 keeps the all-zero border rows ((0, 0) is always among them); min_conf = 1 drops them
        assert confs[0] == 0 and confs[1] == 1
        assert (ref[f"{name}/{mat}/{b}/0/matches"] == 0).all(1).any()


def test_oracle_tie_rules():
    """First-index maxima, NaN maximal, ties among the survivors by ascending i, the last row and column ignored."""
    nan = float("nan")
    s = torch.tensor([[0.0, 0.0, 0.0, 0.0, 9.0],
                      [0.0, 0.5, 0.0, 0.0, 0.0],
                      [0.0, 0.0, 0.0, 0.5, 0.0],
                      [nan, 0.0, 0.0, 0.0, 0.0],
                      [9.0, 9.0, 9.0, 9.0, 9.0]])
    m, v = matches_oracle.matches_list(s)
    # row 0: argmax 0 (first of the zeros), but column 0's maximum is the NaN of row 3; rows 1 and 2 tie at 0.5
    assert m.tolist() == [[1, 1], [2, 3]] and v.tolist() == [0.5, 0.5]
    m, _ = matches_oracle.matches_list(s, min_conf=math.exp(0.5))
    assert m.tolist() == []
    m, _ = matches_oracle.matches_list(s, min_conf=1.6)
    assert m.tolist() == [[1, 1], [2, 3]]


@pytest.mark.parametrize("bad", [torch.zeros(4, 4), torch.zeros(1, 4, 5), torch.zeros(1, 1, 1), torch.zeros(2, 3, 3, 3),
                                 torch.zeros(1, 4098, 4098, dtype=torch.bool)])
def test_mutual_matches_rejects_bad_shapes(bad):
    with pytest.raises(ValueError):
        mutual_matches(bad)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float16, torch.int32])
def test_mutual_matches_rejects_bad_dtypes(dtype):
    with pytest.raises(ValueError, match="float32"):
        mutual_matches(torch.zeros(1, 5, 5, dtype=dtype))


def test_mutual_matches_rejects_cpu_tensors():
    with pytest.raises(ValueError, match="CUDA"):
        mutual_matches(torch.zeros(2, 5, 5))


@pytest.mark.parametrize("min_conf", [float("nan"), float("inf"), -float("inf"), 1e300, "high", None])
def test_mutual_matches_rejects_bad_min_conf(min_conf):
    with pytest.raises(ValueError, match="min_conf"):
        mutual_matches(torch.zeros(1, 5, 5), min_conf)


def test_get_matches_list_rejects_batches():
    with pytest.raises(ValueError, match="batch size 1"):
        featureMatcher().get_matches_list(torch.zeros(2, 5, 5))


def test_matcher_keeps_reference_names_and_method():
    model = MickeyRelativePose(mickey_cfg("vits", 2, 8))
    matcher = model.compute_matches.matcher
    assert isinstance(matcher, featureMatcher) and callable(matcher.get_matches_list)
    assert set(synthetic_state_dict(mickey_cfg("vits", 2, 8), seed=0)) == set(model.state_dict())
