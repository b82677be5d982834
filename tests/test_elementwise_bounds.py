"""CPU test of the element-wise checking helpers (tests/elementwise.py): each bound accepts a correct fp32 computation
of its operation, and each kind of mutation the GPU stage checks use is rejected on the same inputs."""
import pytest
import torch
import torch.nn.functional as F

from tests import elementwise as ew


def _half(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).clamp(-60, 60).half()


@pytest.mark.parametrize("K", [64, 768, 3072, 9 * 512])
@pytest.mark.parametrize("scale", [1.0, 60.0])
def test_gemm_bound_accepts_fp32_products_and_rejects_a_dropped_k_chunk(K, scale):
    M, N = 256, 128
    a, b = _half(M, K, scale=scale, seed=1), _half(N, K, scale=scale, seed=2)
    bias = torch.randn(N, dtype=torch.float64, generator=torch.Generator().manual_seed(3)).float()
    got = (a.float() @ b.float().t() + bias).relu()                       # fp32, blocked CPU accumulation
    A, B = a.double(), b.double()
    pre = A @ B.t() + bias.double()
    ref = pre.relu()
    bound = ew.gemm_acc_bound(K, A.abs() @ B.abs().t()) + ew.epilogue_terms(pre, bias.double()) + ew.out_rounding(ref, False)
    # one 64-wide K chunk dropped from the tile holding rows 128..255 (its second M-tile)
    k0 = (K // 64 - 1) * 64
    drop = (pre[128:] - A[128:, k0:k0 + 64] @ B[:, k0:k0 + 64].t()).relu()
    muts = [ew.Mutation("K chunk dropped", (slice(128, 256), slice(0, N)), drop), ew.row_chunk_swap(ref, 200, 32)]
    r = ew.check(f"gemm K={K}", got, ref, bound, ew.matrix_where(tiles=ew.GemmTiles(M, N)), muts)
    assert 0 <= r <= 1
    if scale == 1.0:                                                   # fp16 output of the same GEMM (EPI_STORE_H)
        got_h = got.half()
        assert ew.check("gemm fp16 out", got_h, ref, bound + ew.out_rounding(ref, True), mutations=muts) <= 1


def test_conv_bound_rejects_a_shifted_tap_a_neighbouring_image_and_pe_row():
    """3x3 conv as 9 row-shifted GEMMs over a zero-padded NHWC grid, fp32, with the sine PE added after the ReLU."""
    n_img, h2, w2, cin, cout = 3, 8, 7, 128, 64
    per = h2 * w2
    x = _half(n_img, h2, w2, cin, seed=4).double()
    x[:, 0] = 0; x[:, -1] = 0; x[:, :, 0] = 0; x[:, :, -1] = 0
    A = x.reshape(-1, cin)
    W = _half(cout, 9 * cin, scale=0.05, seed=5).double()
    pe = torch.randn(per, cout, dtype=torch.float64, generator=torch.Generator().manual_seed(6))
    shifts = [(ky - 1) * w2 + (kx - 1) for ky in range(3) for kx in range(3)]
    R = A.shape[0]

    def shifted(s):
        out = torch.zeros_like(A)
        lo, hi = max(0, -s), min(R, R - s)
        out[lo:hi] = A[lo + s:hi + s]
        return out

    def conv(A_of, Wm):
        return sum(A_of(t) @ Wm[:, t * cin:(t + 1) * cin].t() for t in range(9))

    pre = conv(lambda t: shifted(shifts[t]), W)
    absp = conv(lambda t: shifted(shifts[t]).abs(), W.abs())
    pos = torch.arange(R) % per
    valid = ((pos // w2 >= 1) & (pos // w2 <= h2 - 2) & (pos % w2 >= 1) & (pos % w2 <= w2 - 2))[:, None]
    ref = torch.where(valid, pre.relu() + pe[pos], torch.zeros_like(pre))
    got = torch.where(valid, (conv(lambda t: shifted(shifts[t]).float(), W.float())).relu() + pe[pos].float(), 0.0)
    bound = ew.gemm_acc_bound(9 * cin, absp) + ew.epilogue_terms(pre, pe[pos]) + ew.out_rounding(ref, False)
    m = per + 3 * w2 + 3                                               # image 1, y 3, x 3
    rows = slice(m, m + 1)
    tap = 4
    off_tap = (pre[m] - shifted(shifts[tap])[m] @ W[:, tap * cin:(tap + 1) * cin].t()
               + shifted(shifts[tap] + w2)[m] @ W[:, tap * cin:(tap + 1) * cin].t()).relu() + pe[pos[m]]
    muts = [ew.Mutation("tap 4 one padded row off", (rows, slice(None)), off_tap[None]),
            ew.Mutation("token of the neighbouring image", (rows, slice(None)), ref[m + per][None]),
            ew.Mutation("PE row of the neighbouring position", (rows, slice(None)), (pre[m].relu() + pe[pos[m] + 1])[None])]
    where = ew.matrix_where(ew.Rows("padded", per, w2), ew.GemmTiles(R, cout))
    assert ew.check("conv", got, ref, bound, where, muts) <= 1


@pytest.mark.parametrize("D,scale", [(128, 1.0), (768, 8.0), (1024, 30.0)])
def test_layernorm_bound_accepts_fp32_layernorm(D, scale):
    g = torch.Generator().manual_seed(D)
    x = (torch.randn(300, D, generator=g, dtype=torch.float64) * scale + 3.0).float()
    gamma, beta = torch.randn(D, generator=g).float(), torch.randn(D, generator=g).float()
    got = F.layer_norm(x, (D,), gamma, beta, 1e-6).half()
    ref, b = ew.ln_bound(x.double(), 0.0, gamma.double(), beta.double(), 1e-6)
    b = b + ew.out_rounding(ref, True)
    assert ew.check("layernorm", got, ref, b, mutations=[ew.row_chunk_swap(ref, 10, 64)]) <= 1
    # LayerNorm epilogue of a K = 256 GEMM (inputs with accumulation error)
    a, w = _half(300, 256, seed=7), _half(D, 256, scale=0.1, seed=8)
    acc = a.float() @ w.float().t()
    got = F.layer_norm(acc, (D,), gamma, beta, 1e-5)
    A, Wd = a.double(), w.double()
    ref, b = ew.ln_bound(A @ Wd.t(), ew.gemm_acc_bound(256, A.abs() @ Wd.abs().t()), gamma.double(), beta.double(), 1e-5)
    assert ew.check("gemm + layernorm", got, ref, b + ew.out_rounding(ref, False), mutations=[ew.row_chunk_swap(ref, 3, 0)]) <= 1


@pytest.mark.parametrize("T,scale", [(211, 1.5), (1939, 1.5), (300, 6.0)])
def test_attention_bound_accepts_fp32_attention_with_fp16_p(T, scale):
    g = torch.Generator().manual_seed(T)
    q, k, v = ((torch.randn(3, T, 64, generator=g) * scale).half() for _ in range(3))
    s = (q.float() @ k.float().transpose(-1, -2)) * 0.125
    p = torch.exp(s - s.amax(-1, keepdim=True))
    got = ((p.half().float() @ v.float()) / p.sum(-1, keepdim=True)).half()
    ref, bound = ew.attention_ref_bound(q.double(), k.double(), v.double())
    muts = [ew.Mutation("query 5 attends to the neighbouring image", (0, slice(5, 6)), ref[1, 5:6]),
            ew.Mutation("32-column chunk of the next query", (1, slice(7, 8), slice(32, 64)), ref[1, 8:9, 32:64])]
    assert ew.check("attention", got, ref, bound, mutations=muts) <= 1


def test_split_descriptor_mutation_is_rejected():
    d = F.normalize(torch.randn(50, 128, generator=torch.Generator().manual_seed(9)), dim=-1)
    hi, lo = ew.split_hi_lo(d)
    role0 = torch.cat([hi, lo, hi], -1)
    assert torch.equal(hi.double() + lo.double(), (hi.float() + lo.float()).double())
    assert float((hi.double() + lo.double() - d.double()).abs().max()) <= 2.0 ** -22
    swapped = torch.cat([lo, hi, hi], -1)
    assert ew.check_exact("dscx", role0, role0.clone(), mutations=[ew.Mutation("hi and lo swapped", (slice(None),), swapped)]) == 0


def test_check_reports_the_tile_and_round_of_a_wrong_element():
    """A wrong element in a persistent launch is reported with its image, position, tile and round."""
    R, w2, per = 135680, 40, 2120
    tiles = ew.GemmTiles(R, 512, groups=4, group_fast=True)
    assert tiles.persistent and tiles.tiles == 16960
    ref = torch.zeros(4, 2 * 512, dtype=torch.float64)
    got = ref.clone()
    got[2, 600] = 1.0
    where = ew.matrix_where(ew.Rows("padded", per, w2), tiles, group_width=512, row_offset=130000)
    with pytest.raises(AssertionError) as ei:
        ew.check("T1", got, ref, 1e-3, where)
    msg = str(ei.value)
    t = tiles.tile_of(130002, 88, 1)
    assert t["tile"] == ((130002 // 128) * 4 + 1) * 4 + 0 and f"round {t['tile'] // 132}" in msg, msg
    assert "1 of 4096 elements" in msg and "image 61" in msg and "group 1, column 88" in msg, msg
