"""mk_mutual_matches (featureMatcher.get_matches_list in CUDA) against the CPU oracle on the same fp32 matrices: the
engine's own final_scores / scores at C2 (one ViT-S pair) and C3 (32 ViT-B pairs), padded and contiguous, and planted
matrices for every tie and edge rule.  Integer outputs, so every comparison is exact."""
import math

import pytest
import torch

from mickey_b200.config import mickey_cfg
from mickey_b200.matches import mutual_matches, mutual_matches_raw
from mickey_b200.model import build_model
from mickey_b200.weights import synthetic_checkpoint
from oracle.matches_oracle import matches_list
from tests.common import synthetic_pair

pytestmark = pytest.mark.gpu
DEV = "cuda"
MIN_CONFS = (0.0, 1.5, math.exp(0.5))


def check(scores, min_conf=0.0):
    """Run the kernel on scores [B, N, N] (CUDA, any layout it accepts) and compare every pair with the oracle."""
    m, v, c = mutual_matches_raw(scores, min_conf)
    m, v, c = m.cpu(), v.cpu(), c.cpu()
    host = scores.cpu()
    W = scores.shape[1] - 1
    assert m.shape == (scores.shape[0], W, 2) and v.shape == (scores.shape[0], W)
    for b in range(scores.shape[0]):
        rm, rv = matches_list(host[b], min_conf)
        n = int(c[b])
        assert n == len(rm), (b, n, len(rm))
        assert torch.equal(m[b, :n].long(), rm), b
        assert torch.equal(v[b, :n], rv), b
        assert bool((m[b, n:] == -1).all()) and bool((v[b, n:] == 0).all()), b
    return m, v, c


def padded(t, pitch):
    """t [B, N, N] as the engine lays it out: a [B, N, pitch] buffer viewed as [:, :, :N]."""
    B, N, _ = t.shape
    buf = torch.full((B, N, pitch), float("nan"), device=t.device)   # the padding must never be read as a candidate
    buf[:, :, :N] = t
    return buf[:, :, :N]


@pytest.fixture(scope="module")
def engine_outputs():
    import os
    os.environ.setdefault("MICKEY_SYNTHETIC_BACKBONE", "1")
    out = {}
    for name, variant, it_m, it_r, B in (("c2", "vits", 8, 64, 1), ("c3", "vitb", 16, 64, 32)):
        cfg = mickey_cfg(variant, it_m, it_r)
        model = build_model(cfg, synthetic_checkpoint(cfg, seed=0, with_backbone=True))
        data = {k: v.to(DEV) for k, v in synthetic_pair(B, 720, 540, seed=21).items()}
        torch.manual_seed(0)
        model(data)
        out[name] = (model, data)
    return out


@pytest.mark.parametrize("case", ["c2", "c3"])
@pytest.mark.parametrize("key", ["final_scores", "scores"])
@pytest.mark.parametrize("min_conf", MIN_CONFS)
def test_engine_outputs(engine_outputs, case, key, min_conf):
    model, data = engine_outputs[case]
    s = data[key]
    assert s.stride(1) == 1952 or s.is_contiguous()          # the engine's padded layout at 720x540 (pitch 1952)
    m, _, c = check(s, min_conf)
    if min_conf == 0.0:
        assert bool((c > 0).all())
    if min_conf == 0.0 and key == "final_scores":
        # the border keypoints' zero rows and columns make (0, 0) a match with score 0 in every pair
        assert all(((m[b, :int(c[b])] == 0).all(1)).any() for b in range(len(c)))
    check(s.contiguous(), min_conf)
    check(padded(s, 1952), min_conf)


def test_matcher_get_matches_list_is_the_oracle(engine_outputs):
    model, data = engine_outputs["c3"]
    matcher = model.compute_matches.matcher
    for b in (0, 17, 31):
        got = matcher.get_matches_list(data["final_scores"][b].unsqueeze(0))
        assert got.dtype == torch.int64 and got.device.type == "cuda"
        assert torch.equal(got.cpu(), matches_list(data["final_scores"][b].cpu())[0])
    lists, scores = model.mutual_matches(data["final_scores"], 0.0)
    assert len(lists) == len(scores) == 32
    for b in range(32):
        rm, rv = matches_list(data["final_scores"][b].cpu())
        assert torch.equal(lists[b].cpu(), rm) and torch.equal(scores[b].cpu(), rv)


def test_repeated_calls_are_byte_identical(engine_outputs):
    _, data = engine_outputs["c3"]
    first = [t.clone() for t in mutual_matches_raw(data["final_scores"])]
    for _ in range(3):
        again = mutual_matches_raw(data["final_scores"])
        assert all(torch.equal(a, b) for a, b in zip(first, again))


def planted(N, seed, B=1):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, N, N, generator=g)


@pytest.mark.parametrize("layout", ["contiguous", "padded"])
def test_planted_rules(layout):
    N = 300
    s = planted(N, 1, B=3)
    s[0, 5] = 0.0                                   # an all-zero row
    s[0, :, 7] = 0.0
    s[0, 9, [3, 40, 200]] = 2.0                     # tied maxima within one row: the first column wins
    s[0, [10, 100, 250], 60] = 3.0                  # tied maxima of one column in three row strips (64 rows each)
    s[1, 20, 21] = s[1, 30, 31] = s[1, 40, 41] = 5.0   # tied scores among the survivors: ordered by ascending i
    s[1, 50, 51] = float("nan")                     # NaN is maximal in its row and column, and never a match
    s[1, 52, 53] = float("nan")
    s[1, 60, 53] = float("nan")                     # two NaNs in one column: the first row wins
    s[2, :, 150] = float("-inf")
    s[2, 70] = -1.0
    s[2, :, 71] = -2.0
    s[2, 70, 71] = -0.0                             # mutual matches scored -0.0 (row 70) and +0.0 (row 80): equal scores,
    s[2, 80] = -1.0                                 # so row 70 comes first
    s[2, :, 81] = -2.0
    s[2, 80, 81] = 0.0
    s[2, N - 1, :] = 10.0                           # the last row and column are not candidates
    s[2, :, N - 1] = 10.0
    s = s.to(DEV)
    if layout == "padded":
        s = padded(s, 304)
    for c in (0.0, 1.5, math.exp(0.5), -1.0):
        m, _, cnt = check(s, c)
    m, v, cnt = check(s)
    rows1 = m[1, :3, 0].tolist()
    assert rows1 == [20, 30, 40] and v[1, :3].tolist() == [5.0] * 3


@pytest.mark.parametrize("N", [2, 3, 33, 64, 65, 129, 1938, 2049, 4097])
def test_sizes(N):
    s = planted(N, N, B=2)
    s[1, : N // 2] = 0.0
    s = s.to(DEV)
    check(s)
    check(s, 1.5)
    if N % 4 != 0:
        check(padded(s, (N + 31) // 32 * 32))


def test_all_zero_matrix_and_batch_32():
    s = torch.zeros(32, 65, 65, device=DEV)
    m, v, c = check(s)
    assert c.tolist() == [1] * 32 and m[:, 0].tolist() == [[0, 0]] * 32     # (0, 0) is the only mutual pair
    _, _, c = check(s, 1.0)                                                  # exp(0) = 1 is not > 1
    assert c.tolist() == [0] * 32


def test_exp_threshold_boundary():
    """The threshold is on exp(max) rounded to fp32: a maximum of exactly 0.5 does not pass min_conf = e^0.5."""
    s = torch.zeros(1, 5, 5, device=DEV)
    s[0, 1, 1] = 0.5
    s[0, 2, 2] = 0.5000001
    m, _, c = check(s, math.exp(0.5))
    assert m[0, :int(c[0])].tolist() == [[2, 2]]


def test_odd_layouts_are_copied():
    s = planted(70, 5, B=2).to(DEV)
    check(s.transpose(1, 2))                         # last dimension not contiguous: read from a contiguous copy
    base = torch.zeros(2, 80, 70, device=DEV)        # pairs further apart than N row pitches
    base[:, :70] = s
    check(base[:, :70, :])
    lists, _ = mutual_matches(s.transpose(1, 2))
    assert torch.equal(lists[0].cpu(), matches_list(s[0].t().cpu())[0])
