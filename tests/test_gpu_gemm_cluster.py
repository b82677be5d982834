"""The persistent GEMM on two-CTA clusters (M-adjacent tiles share each B tile through TMA multicast) against the same
kernel without pairs, byte for byte: the pairs change which CTA loads which bytes, never the MMAs or their order.

impl "paired" / "unpaired" run the persistent kernel with / without pairs whatever the grid size; "tc" is the default
dispatch, which puts grids of more than 8 tiles per SM on the paired kernel.  Output buffers carry rows beyond M filled
with a sentinel: the rank-1 CTA of the last pair of an odd M-tile count computes a tile wholly beyond M and must store
nothing."""
from unittest import mock

import pytest
import torch

from tests import gpu_util
from tests.gpu_util import gemm
from tests.test_gpu_ops import _rand

pytestmark = pytest.mark.gpu
DEV = "cuda"
IMPLS = {"paired": 3, "unpaired": 4}
SENTINEL = -7.0


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(impl, epi, a, w, M, N, K=None, outs=(), **kw):
    """One launch on fresh copies of the output buffers `outs` (names of tensors in kw); returns the copies."""
    kw = dict(kw)
    for name in outs:
        kw[name] = kw[name].clone()
    with mock.patch.dict(gpu_util.IMPL, IMPLS):
        gemm(epi, a, w, M, N, K, impl=impl, **kw)
    torch.cuda.synchronize()
    return [kw[name] for name in outs]


def _same(epi, a, w, M, N, K=None, outs=(), impls=("unpaired", "paired"), **kw):
    bn = 128 if epi == "LSE" or N % 128 == 0 else 64
    if _m_tiles(M) * -(-N // bn) * kw.get("groups", 1) > 8 * _sms():
        impls += ("tc",)                                     # the default dispatch takes the paired kernel here
    res = {impl: _run(impl, epi, a, w, M, N, K, outs, **kw) for impl in impls}
    ref = res[impls[0]]
    for impl in impls[1:]:
        for name, x, y in zip(outs, ref, res[impl]):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), (impl, name)
    return ref


def _m_tiles(M):
    return -(-M // 128)


@pytest.mark.parametrize("M,N,K,act", [
    (40000, 512, 256, 1),     # 313 M-tiles (odd), 64-row last tile, BN 128, GELU
    (40065, 512, 192, 2),     # 314 M-tiles, a last tile of one row, ReLU
    (50001, 192, 320, 0),     # BN 64 (N % 128 != 0), 391 M-tiles (odd)
])
def test_store_h(M, N, K, act):
    a, w, bias = _rand(M, K, seed=1).half(), _rand(N, K, scale=0.05, seed=2).half(), _rand(N, scale=0.1, seed=3)
    out = torch.full((M + 256, N), SENTINEL, dtype=torch.float16, device=DEV)
    (o,) = _same("STORE_H", a, w, M, N, K, outs=("out_h",), bias=bias, act=act, out_h=out, out_h_ld=N)
    assert bool((o[M:] == SENTINEL).all())
    assert torch.isfinite(o[:M]).all()


@pytest.mark.parametrize("N", [768, 192])
def test_resid_f(N):
    M, K = 46081, 384                                         # 361 M-tiles (odd), a last tile of one row
    a, w = _rand(M, K, seed=4).half(), _rand(N, K, scale=0.05, seed=5).half()
    x = torch.full((M + 128, N), SENTINEL, device=DEV)
    x[:M] = _rand(M, N, seed=6)
    (o,) = _same("RESID_F", a, w, M, N, K, outs=("out_f",), bias=_rand(N, seed=7), gamma=_rand(N, scale=0.1, seed=8),
                 out_f=x, out_f_ld=N)
    assert bool((o[M:] == SENTINEL).all())


@pytest.mark.parametrize("N", [128, 64])
def test_store_f_groups_sharing_a(N):
    """Groups that read the same A: gemm_tile walks the groups between the M-pairs and the N-tiles."""
    R, G, K = 40000, 4, 192                                   # 313 M-tiles (odd) x G
    a = _rand(R, K, seed=9).half()
    w = _rand(G * N, K, scale=0.1, seed=10).half()
    out = torch.full((R + 128, G * N), SENTINEL, device=DEV)
    (o,) = _same("STORE_F", a, w, R, N, K, outs=("out_f",), groups=G, b_row_group_off=N, out_f=out, out_f_ld=G * N,
                 out_f_group_off=N)
    assert bool((o[R:] == SENTINEL).all())


def test_patch():
    n_img, tok, D, K = 33, 1938, 384, 640                     # 63954 rows: 500 M-tiles, 18-row last tile
    M = n_img * tok
    a, w = _rand(M, K, seed=11).half(), _rand(D, K, scale=0.05, seed=12).half()
    pos = _rand(tok, D, seed=13)
    X = torch.full((n_img * (tok + 1), D), SENTINEL, device=DEV)
    (o,) = _same("PATCH", a, w, M, D, K, outs=("out_f",), aux=pos, tok_per_img=tok, out_f=X, out_f_ld=D)
    assert bool((o.reshape(n_img, tok + 1, D)[:, 0] == SENTINEL).all())     # cls rows untouched


@pytest.mark.parametrize("C", [128, 64])
def test_conv3x3_groups_own_a(C):
    """9 taps over a zero-padded NHWC image, groups with their own A columns, bias, fp16 shortcut, ReLU, positional
    table on one group and the pad-row mask; BN 128 and (C = 64) 64."""
    n_img, h2, w2, G = 33, 53, 40, 2                          # 69960 rows: 547 M-tiles (odd), 72-row last tile
    R = n_img * h2 * w2
    a = _rand(R, G * C, seed=14).half()
    w = _rand(G * C, 9 * C, scale=0.02, seed=15).half()
    taps = [(ky - 1) * w2 + (kx - 1) for ky in range(3) for kx in range(3)]
    out = torch.full((R + 128, G * C), SENTINEL, dtype=torch.float16, device=DEV)
    (o,) = _same("CONV", a, w, R, C, taps=taps, chunks_per_tap=C // 64, outs=("out_h",),
                 groups=G, a_col_group_off=C, b_row_group_off=C, bias=_rand(G * C, seed=16), bias_group_off=C,
                 res_h=_rand(R, G * C, seed=17).half(), res_h_ld=G * C, res_h_group_off=C, act=2,
                 aux=_rand(h2 * w2, C, seed=18), aux_group_mask=1, pad_h2=h2, pad_w2=w2,
                 out_h=out, out_h_ld=G * C, out_h_group_off=C)
    assert bool((o[R:] == SENTINEL).all())


def test_conv3x3_bn64():
    """BN 64 on a 9-tap convolution: 192 output channels per group."""
    n_img, h2, w2, Cin, Cout = 33, 53, 40, 128, 192
    R = n_img * h2 * w2
    a = _rand(R, Cin, seed=19).half()
    w = _rand(Cout, 9 * Cin, scale=0.02, seed=20).half()
    taps = [(ky - 1) * w2 + (kx - 1) for ky in range(3) for kx in range(3)]
    out = torch.full((R + 128, Cout), SENTINEL, dtype=torch.float16, device=DEV)
    (o,) = _same("CONV", a, w, R, Cout, taps=taps, chunks_per_tap=Cin // 64, outs=("out_h",), bias=_rand(Cout, seed=21),
                 act=2, pad_h2=h2, pad_w2=w2, out_h=out, out_h_ld=Cout)
    assert bool((o[R:] == SENTINEL).all())


def test_matcher_pass1_odd_m_tiles():
    """EPI_LSE with per-group A (one group per image pair, A rows offset by n_valid) and 15 M-tiles per group: the
    phantom tile of each group's last pair would write the column partials of a 16th M-tile if its epilogue ran, over
    the next group's first slots, and past the last group's into the 4 spare slots."""
    B, N = 5, 1900
    npad = (N + 127) // 128 * 128
    a0, a1 = _rand(B * N, 384, scale=0.05, seed=22).half(), _rand(B * N, 384, scale=0.05, seed=23).half()
    pr = torch.full((B, npad // 64, npad, 2), SENTINEL, device=DEV)
    pc = torch.full((B * (npad // 32) + 4, npad, 2), SENTINEL, device=DEV)  # 4 slots per M-tile and group, + 4 spare
    pr_o, pc_o = _same("LSE", a0, a1, N, N, 384, outs=("part_row", "part_col"), groups=B, a_row_group_off=N,
                       b_row_group_off=N, n_valid=N, inv_temp=10.0, part_ld=npad, part_row=pr, part_col=pc)
    assert bool((pc_o[B * (npad // 32):] == SENTINEL).all())


@pytest.mark.parametrize("M", [1100, 129, 1])
def test_grid_below_resident_clusters(M):
    """A handful of tile pairs (fewer than the clusters that fit on the device), an odd M-tile count, a one-row M."""
    N, K = 256, 512
    a, w = _rand(M, K, seed=24).half(), _rand(N, K, scale=0.05, seed=25).half()
    out = torch.full((M + 128, N), SENTINEL, device=DEV)
    (o,) = _same("STORE_F", a, w, M, N, K, outs=("out_f",), impls=("unpaired", "paired"), out_f=out, out_f_ld=N)
    assert bool((o[M:] == SENTINEL).all())
    ref = a.float() @ w.float().t()
    assert float((o[:M] - ref).abs().max()) < 1e-3 * float(ref.abs().max())
