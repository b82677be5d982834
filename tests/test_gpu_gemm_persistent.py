"""The persistent wgmma GEMM (grids of more than 8 tiles per SM; 1056 tiles on a 132-SM H100) on the paths the other GEMM
tests do not reach: 64-wide tiles, the matcher's first pass, and groups that share A (the group-fast tile order)."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.common import rel_err
from tests.gpu_util import gemm
from tests.test_gpu_ops import _dual_softmax_ref, _matcher, _rand

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _more_than_8_per_sm(tiles):
    assert tiles > 8 * torch.cuda.get_device_properties(0).multi_processor_count, tiles


def test_persistent_bn64_store_h():
    """N % 128 != 0 -> 64-wide tiles on the 6-stage persistent ring, with an M tail."""
    M, N, K = 50001, 192, 320                                   # 391 x 3 = 1173 tiles, K = 5 chunks
    _more_than_8_per_sm(-(-M // 128) * (N // 64))
    a, w, bias = _rand(M, K, seed=60).half(), _rand(N, K, scale=0.05, seed=61).half(), _rand(N, scale=0.1, seed=62)
    out = torch.zeros(M, N, dtype=torch.float16, device=DEV)
    gemm("STORE_H", a, w, M, N, K, bias=bias, act=1, out_h=out, out_h_ld=N)
    assert rel_err(out, F.gelu(a.float() @ w.float().t() + bias)) < 2e-3


def test_persistent_groups_sharing_a():
    """Four groups reading the same A columns (a_col_group_off = a_row_group_off = 0): gemm_tile walks the groups between
    the M-tiles and the N-tiles, over several rounds of the persistent grid."""
    R, G, K, N = 40000, 4, 192, 128                             # 313 x 1 x 4 = 1252 tiles
    _more_than_8_per_sm(-(-R // 128) * G)
    a = _rand(R, K, seed=63).half()
    w = _rand(G * N, K, scale=0.1, seed=64).half()
    out = torch.full((R, G * N), 7.0, device=DEV)
    gemm("STORE_F", a, w, R, N, K, groups=G, b_row_group_off=N, out_f=out, out_f_ld=G * N, out_f_group_off=N)
    for g in range(G):
        assert rel_err(out[:, g * N:(g + 1) * N], a.float() @ w[g * N:(g + 1) * N].float().t()) < 1e-5, g


def test_persistent_matcher_pass1():
    """EPI_LSE on a persistent grid (5 pairs of 1938 keypoints: 1280 tiles), then the reduce and EPI_DUAL."""
    B, N, T = 5, 1938, 0.1
    _more_than_8_per_sm(B * (-(-N // 128)) ** 2)
    d0 = F.normalize(_rand(B, N, 128, seed=65), dim=-1)
    d1 = F.normalize(_rand(B, N, 128, seed=66), dim=-1)
    s0, s1 = torch.rand(B, N, device=DEV), torch.rand(B, N, device=DEV)
    dust = torch.tensor([1.0], device=DEV)
    sc, _, fin, lr, lc = _matcher(d0, d1, s0, s1, T, dust)
    ref, S = _dual_softmax_ref(d0, d1, T, 1.0)
    lse_r = torch.logsumexp(torch.cat([S, torch.full_like(S[:, :, :1], 1.0)], 2), 2) / math.log(2)
    lse_c = torch.logsumexp(torch.cat([S, torch.full_like(S[:, :1, :], 1.0)], 1), 1) / math.log(2)
    assert float((lr[:, :N].double() - lse_r).abs().max()) < 1e-4 and float((lc[:, :N].double() - lse_c).abs().max()) < 1e-4
    assert rel_err(sc, ref) < 1e-4
    assert rel_err(fin, ref * s0[:, :, None].double() * s1[:, None, :].double()) < 1e-4
