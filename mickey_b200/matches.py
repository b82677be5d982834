"""MicKey's correspondences: featureMatcher.get_matches_list (lib/models/MicKey/modules/utils/feature_matcher.py:19-46) on
the GPU, batched, through mk_mutual_matches (csrc/matches.cu).

A match (i, j) is a mutual nearest neighbour of the score matrix with the last row and column dropped (as the reference
does), whose exp(score) exceeds min_conf.  The lists are sorted by score, descending; equal scores (the border keypoints'
zero rows make them common) are ordered by ascending i, which the reference's unstable sort leaves open.
"""
from __future__ import annotations

import math
from typing import List, Tuple

import numpy as np
import torch

from . import _lib

MAX_N = 4097          # N - 1 candidates are sorted in one block's shared memory


def _check_min_conf(min_conf) -> float:
    try:
        v = float(min_conf)
    except (TypeError, ValueError):
        raise ValueError(f"min_conf must be a real number, got {min_conf!r}") from None
    if not math.isfinite(v) or abs(v) > float(np.finfo(np.float32).max):
        raise ValueError(f"min_conf must be finite in fp32, got {min_conf!r}")
    return v


def _check_scores(scores) -> torch.Tensor:
    if not torch.is_tensor(scores):
        raise ValueError(f"scores must be a torch tensor, got {type(scores).__name__}")
    if scores.dim() != 3 or scores.shape[1] != scores.shape[2]:
        raise ValueError(f"scores must be [B, N, N], got {tuple(scores.shape)}")
    B, N = scores.shape[0], scores.shape[1]
    if B < 1 or not 2 <= N <= MAX_N:
        raise ValueError(f"scores [B, N, N] needs B >= 1 and 2 <= N <= {MAX_N}, got {tuple(scores.shape)}")
    if scores.dtype != torch.float32:
        raise ValueError(f"scores must be float32 (the matcher's output), got {scores.dtype}")
    if scores.device.type != "cuda":
        raise ValueError(f"scores must be on a CUDA device (mickey_b200 has no CPU path), got {scores.device}")
    return scores


def mutual_matches_raw(scores: torch.Tensor, min_conf: float = 0.0):
    """One launch pair for all B matrices.  Returns (matches int32 [B, N-1, 2], match_scores fp32 [B, N-1], count int32
    [B]), all on the scores' device; rows from count[b] on are (-1, -1) / 0.  A view whose last dimension is contiguous and
    whose pairs lie N row pitches apart (the engine's padded [B, N, pitch][:, :, :N] views, contiguous tensors) is read in
    place; any other layout is copied to a contiguous tensor first."""
    min_conf = _check_min_conf(min_conf)
    scores = _check_scores(scores)
    B, N = scores.shape[0], scores.shape[1]
    scores, pitch = _lib.pitched(scores)
    lib = _lib.load()
    dev = scores.device
    W = N - 1
    with torch.cuda.device(dev):
        matches = torch.empty(B, W, 2, dtype=torch.int32, device=dev)
        match_scores = torch.empty(B, W, dtype=torch.float32, device=dev)
        count = torch.empty(B, dtype=torch.int32, device=dev)
        ws = _lib.workspace(lib.mk_mutual_matches_ws_bytes(B, N), dev, "mk_mutual_matches_ws_bytes")
        _lib.check(lib.mk_mutual_matches(_lib.ptr(scores), pitch, B, N, min_conf, _lib.ptr(matches), _lib.ptr(match_scores),
                                         _lib.ptr(count), _lib.ptr(ws), ws.numel(), _lib.stream(dev)), "mk_mutual_matches")
    return matches, match_scores, count


def mutual_matches(scores: torch.Tensor, min_conf: float = 0.0) -> Tuple[List[torch.Tensor], List[torch.Tensor]]:
    """get_matches_list of every pair of scores [B, N, N] fp32 (CUDA): a list of B int64 [M_b, 2] tensors (i, j) and a
    list of their B fp32 [M_b] scores, on the scores' device.  One device-to-host copy (the counts)."""
    matches, match_scores, count = mutual_matches_raw(scores, min_conf)
    counts = count.cpu().tolist()
    return ([matches[b, :c].long() for b, c in enumerate(counts)],
            [match_scores[b, :c] for b, c in enumerate(counts)])
