"""CPU oracle of MicKey's correspondences: featureMatcher.get_matches_list restated in plain PyTorch.

Test infrastructure, like oracle/mickey_oracle.py: only tests/ and tools/ import it, mickey_b200 never does.  Pinned to the
live reference by tests/golden/reference_matches_720x540.npz (tests/golden/make_matches_fixture.py).
"""
from __future__ import annotations

from typing import Tuple

import torch

Tensor = torch.Tensor


def matches_list(scores: Tensor, min_conf: float = 0.0) -> Tuple[Tensor, Tensor]:
    """lib/models/MicKey/modules/utils/feature_matcher.py:19-46 (featureMatcher.get_matches_list) on one pair, scores
    [1, N, N] or [N, N].  Returns (matches int64 [M, 2] = (i, j), their scores scores[i, j] [M]).

    * The last row and column are dropped (:24, `scores[:, :-1, :-1]`, written for a matrix that still held the dustbin;
      the reference calls it on final_scores, which has none, and so does this).
    * Row and column maxima follow torch.max(dim): the first maximal index wins, and a NaN counts as maximal.
    * (i, j) is kept when j is row i's argmax and i is column j's argmax (:26) and exp(max) > min_conf (:29-30).  exp is
      taken in float64 and rounded to the scores' dtype (the correctly rounded exp), then compared in that dtype as torch
      compares a tensor with a Python scalar; a NaN maximum never passes.  With min_conf = 0 every mutual pair passes,
      all-zero rows included.
    * The list is sorted by score, descending (:44).  The reference's torch.sort is not stable, so it leaves the order of
      equal scores open; here equal scores are ordered by ascending i (a stable sort of the row-ordered list)."""
    s = scores.reshape(scores.shape[-2], scores.shape[-1])[:-1, :-1]
    max0, max1 = s.max(1), s.max(0)
    idx0, idx1 = max0.indices, max1.indices
    rows = torch.arange(s.shape[0], device=s.device)
    mutual = rows == idx1[idx0]
    thr = torch.tensor(min_conf, dtype=s.dtype, device=s.device)
    valid = mutual & (torch.exp(max0.values.double()).to(s.dtype) > thr)
    i, j = rows[valid], idx0[valid]
    vals = s[i, j]
    order = torch.sort(vals, descending=True, stable=True).indices
    return torch.stack([i, j], 1)[order], vals[order]
