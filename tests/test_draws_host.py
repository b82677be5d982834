"""CPU checks of the draw restatements in tests/draws.py, and the failure contract decided by torch itself."""
import numpy as np
import pytest
import torch

from mickey_b200.config import mickey_cfg
from oracle import mickey_oracle as mo
from tests import draws


def _philox_np(c0, c1, c2, c3, seed):
    from tests.test_gpu_ops import _philox4x32_7
    return _philox4x32_7(c0, c1, c2, c3, seed)


@pytest.mark.parametrize("seed", [0, 1, 0x1234567887654321, 0xFFFFFFFFFFFFFFFF, 0x9E3779B97F4A7C15 ^ 77])
def test_philox_matches_numpy_restatement(seed):
    g = np.random.default_rng(seed & 0xFFFF)
    c = [g.integers(0, 2 ** 32, 4096, dtype=np.uint64).astype(np.uint32) for _ in range(4)]
    c[0][:4] = [0, 1, 0xFFFFFFFF, 0x80000000]
    want = _philox_np(*c, seed)
    got = draws.philox(*(torch.from_numpy(x.astype(np.int64)) for x in c), seed)
    for w, x in zip(want, got):
        assert np.array_equal(w.astype(np.int64), x.numpy())


def test_outer_keys_match_numpy_restatement():
    """The fp64 keys of two streams of different Philox groups against a direct numpy evaluation (the formula of
    test_outer_sampler_is_topk_of_the_race); torch's and numpy's log1p may differ in the last bit."""
    seed, b = 0x0123456789ABCDEF, 3
    p = torch.rand(5000, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    p[::7] = 0
    keys = dict(draws.outer_keys(p, seed, b, [2, 9], chunk=1024))
    e = np.arange(5000, dtype=np.uint32)
    for s in (2, 9):
        sg, j = divmod(s, 8)
        w = _philox_np(e, np.uint32(0x5bd1e995), np.uint32(sg), np.uint32(b), seed)[j >> 1]
        prefix = (w >> np.uint32((j & 1) * 16)) & np.uint32(0xffff)
        low = _philox_np(e, np.uint32(0x2545F491), np.uint32(s), np.uint32(b), seed)[0]
        u = (prefix.astype(np.float64) + (low.astype(np.float64) + 0.5) * 2.0 ** -32) * 2.0 ** -16
        want = np.where(p.numpy() > 0, p.numpy() / -np.log1p(-u), 0.0)
        assert np.allclose(keys[s].numpy(), want, rtol=4e-16, atol=0)


def test_band_check_rejects_planted_mutations():
    """The band check accepts the fp64 draw and draws that differ only inside the band, and rejects: the 2049th cell
    swapped in for a true top-2048 cell, and a drawn cell at a row end shifted to the next row's first cell."""
    N, n_s = 100, 2048
    p = torch.rand(N * N, generator=torch.Generator().manual_seed(1), dtype=torch.float64) ** 4
    key = dict(draws.outer_keys(p, 77, 0, [5]))[5]
    ref = draws.reference_draw(key, n_s)
    assert draws.band_check(ref, key, n_s)["ok"]
    order = torch.argsort(key, descending=True)
    # a near-tie at the boundary is excused: nudge the 2049th key into the band and swap it with the 2048th
    key2 = key.clone()
    key2[order[n_s]] = key[order[n_s - 1]] * (1 - 0.5 * draws.BAND)
    swapped = ref.clone()
    swapped[swapped == order[n_s - 1]] = order[n_s]
    assert draws.band_check(swapped.sort().values, key2, n_s)["ok"]
    # the 2049th cell in place of the median drawn cell
    bad = ref.clone()
    bad[bad == order[n_s // 2]] = order[n_s]
    r = draws.band_check(bad.sort().values, key, n_s)
    assert not r["ok"] and r["n_bad"] >= 1
    # a draw shifted one cell at a row end
    ends = ref[(ref % N == N - 1) & ~torch.isin(ref + 1, ref)]
    assert ends.numel() > 0
    shifted = ref.clone()
    shifted[shifted == ends[0]] += 1
    assert not draws.band_check(shifted.sort().values, key, n_s)["ok"]


def test_inner_cdf_summation_order():
    """The restated cdf is the kernel's order, not a plain cumulative sum: on weights that span 12 decades the two
    differ, the restatement is exact where the order cannot matter (integer weights), and it is non-decreasing
    within each thread's run."""
    g = torch.Generator().manual_seed(2)
    w = (10.0 ** (-12 * torch.rand(4, 2048, generator=g))).float()
    cdf = draws.inner_cdf(w)
    seq = torch.cumsum(w.double(), 1).float()
    assert not torch.equal(cdf, seq)
    assert float(((cdf.double() - seq.double()).abs() / seq.double()).max()) < 1e-5
    wi = torch.randint(0, 5, (3, 2048), generator=g).float()
    assert torch.equal(draws.inner_cdf(wi), torch.cumsum(wi, 1))
    loc = cdf.reshape(4, 256, 8)
    assert bool((loc[:, :, 1:] >= loc[:, :, :-1]).all())


def test_inner_draw_takes_positive_entries_and_follows_the_guard():
    """Three positive weights: every draw is exactly those three.  One positive weight (the guard's rule): it and the
    two entries after it, cyclically."""
    n = 2048
    w = torch.zeros(2, n)
    w[0, [5, 700, 2047]] = torch.tensor([1.0, 1e-3, 0.3])
    w[1, 2047] = 0.5
    idx, amb = draws.inner_draw(draws.inner_cdf(w), 1234, torch.tensor([0, 0]), torch.tensor([0, 1]), 500)
    assert set(idx[0].sort(1).values.unique(dim=0).reshape(-1).tolist()) == {5, 700, 2047}
    assert bool((idx[0].sort(1).values == torch.tensor([5, 700, 2047])).all())
    assert bool((idx[1] == torch.tensor([2047, 0, 1])).all())


@pytest.mark.parametrize("n", [32, 64, 96, 256, 288, 512, 2048])
def test_loss_inner_cdf_layout(n):
    """The loss kernel's cdf: inner_cdf's exactly when 256 divides the set size; for any other multiple of 32, inner_cdf
    of the weights padded with exact zeros to a multiple of 256 (the trailing threads add nothing).  On weights that
    span 12 decades it is not a plain cumulative sum."""
    g = torch.Generator().manual_seed(n)
    w = (10.0 ** (-12 * torch.rand(6, n, generator=g))).float()
    w[0, ::3] = 0
    cdf = draws.loss_inner_cdf(w)
    assert cdf.shape == (6, n)
    per = -(-n // 256)
    padded = torch.cat([w, torch.zeros(6, 256 * per - n)], 1)
    assert torch.equal(cdf, draws.inner_cdf(padded)[:, :n])
    if n % 256 == 0:
        assert torch.equal(cdf, draws.inner_cdf(w))
    assert not torch.equal(cdf, torch.cumsum(w.double(), 1).float())
    wi = torch.randint(0, 5, (3, n), generator=g).float()
    assert torch.equal(draws.loss_inner_cdf(wi), torch.cumsum(wi, 1))


def _loss_sets(n, rows=16, seed=4):
    """Set weights as the loss sees them: final_scores-like values over four decades, a few exact zeros."""
    g = torch.Generator().manual_seed(seed)
    w = (10.0 ** (-4 * torch.rand(rows, n, generator=g))).float()
    w[torch.rand(rows, n, generator=g) < 0.1] = 0
    return w, torch.arange(rows) // 4, torch.arange(rows) % 4


def test_loss_inner_draw_at_three_with_the_solver_tag_is_the_solver_draw():
    """The C-draw restatement with C = 3 and the solver's Philox tag is the solver's restated draw, element for element
    (the two kernels share the cdf search, the skip and the guard)."""
    w, b_of, s_in = _loss_sets(512)
    cdf = draws.loss_inner_cdf(w)
    got, amb = draws.loss_inner_draw(cdf, 0xC0FFEE, b_of, s_in, 40, 3, tag=draws.INNER_TAG)
    want, amb3 = draws.inner_draw(draws.inner_cdf(w), 0xC0FFEE, b_of, s_in, 40)
    assert torch.equal(got, want) and torch.equal(amb, amb3)


def test_loss_inner_draw_check_rejects_planted_mutations():
    """8 of 64: the check accepts the restatement itself and rejects the solver's tag in place of the loss's, one pick
    replaced by its neighbour, and the skip over drawn mass taken in draw order instead of index order."""
    n, C, IR, seed = 64, 8, 64, 0x5EED
    w, b_of, s_in = _loss_sets(n)
    cdf = draws.loss_inner_cdf(w)
    want, amb = draws.loss_inner_draw(cdf, seed, b_of, s_in, IR, C)
    assert bool((want.sort(-1).values[..., 1:] > want.sort(-1).values[..., :-1]).all())       # C distinct entries
    assert draws.inner_draw_check(want, want, amb)["ok"]
    assert int(amb.sum()) < amb.numel() // 10
    tag, _ = draws.loss_inner_draw(cdf, seed, b_of, s_in, IR, C, tag=draws.INNER_TAG)
    r = draws.inner_draw_check(tag, want, amb)
    assert not r["ok"] and r["n_bad"] > amb.numel() // 2
    clear = torch.nonzero(~amb)
    nb = want.clone()
    r0, h0 = int(clear[0, 0]), int(clear[0, 1])
    nb[r0, h0, 5] = (nb[r0, h0, 5] + 1) % n
    r = draws.inner_draw_check(nb, want, amb)
    assert not r["ok"] and r["n_bad"] == 1
    order, _ = draws.loss_inner_draw(cdf, seed, b_of, s_in, IR, C, skip_in_draw_order=True)
    r = draws.inner_draw_check(order, want, amb)
    assert not r["ok"] and r["n_bad"] >= 1


def test_loss_inner_draw_fills_by_the_guard():
    """5 positive weights of 64, 8 draws: the first five are the positive entries and the guard keeps the other three
    distinct.  With one positive entry the draw is it and the seven entries after it, cyclically."""
    n, C = 64, 8
    w = torch.zeros(2, n)
    pos = [3, 17, 40, 41, 63]
    w[0, pos] = torch.tensor([1.0, 0.2, 0.05, 0.3, 1e-3])
    w[1, 60] = 0.5
    idx, _ = draws.loss_inner_draw(draws.loss_inner_cdf(w), 99, torch.tensor([0, 0]), torch.tensor([0, 1]), 200, C)
    assert bool((idx[0, :, :5].sort(-1).values == torch.tensor(pos)).all())
    assert bool((idx[0].sort(-1).values[:, 1:] > idx[0].sort(-1).values[:, :-1]).all())
    assert bool((idx[1] == torch.tensor([60, 61, 62, 63, 0, 1, 2, 3])).all())


def test_closed_form_law_matches_torch_multinomial():
    """Successive sampling's closed form against torch.multinomial(w, 3) and against the fp64 race top-3 of w / Exp(1)
    (what ATen's multinomial without replacement computes), by chi^2 over 400 k draws; the with-replacement law is
    rejected by the same statistic."""
    w = torch.tensor([1.0, 0.4, 0.2, 0.1, 0.08, 0.05, 0.03, 0.01, 0.005, 0.001], dtype=torch.float64)
    law = draws.law3(w.tolist())
    assert abs(sum(law.values()) - 1) < 1e-12
    n = 400_000
    g = torch.Generator().manual_seed(5)
    mult = torch.multinomial(w.float().expand(n, -1), 3, generator=g).sort(1).values
    race = (w / torch.empty(n, 10, dtype=torch.float64).exponential_(1, generator=g)).topk(3, 1).indices.sort(1).values

    def counts(t):
        u, c = t.unique(dim=0, return_counts=True)
        return {tuple(x): int(k) for x, k in zip(u.tolist(), c.tolist())}

    for t in (mult, race):
        cnt = counts(t)
        assert draws.chi2_pvalue(cnt, law) > 1e-6
        assert draws.chi2_pvalue(cnt, draws.law3_with_replacement(w.tolist())) < 1e-6


@pytest.mark.parametrize("case", sorted(draws.CONTRACT))
def test_failure_contract_table(case):
    """For each edge matrix, whether the reference (through the oracle, which keeps its torch.multinomial calls and its
    try/except) returns the zero pose for the whole batch or a pose; the GPU tests hold the kernels to this table."""
    cfg = mickey_cfg("vits", 2, 8)
    fs = draws.contract_matrix(case)
    kps0, d0, kps1, d1, K = draws.contract_geometry()
    R, t, inl = mo.solve_pose(fs, kps0, d0, kps1, d1, K, K, cfg, generator=torch.Generator().manual_seed(0))
    zero = float(R.abs().max()) == 0 and float(t.abs().max()) == 0 and float(inl.abs().max()) == 0
    assert ("zero" if zero else "pose") == draws.CONTRACT[case]
    if not zero:
        assert bool(torch.isfinite(R).all()) and bool(torch.isfinite(t).all())
    # and it is torch.multinomial itself that decides
    row = fs[draws.CONTRACT_PAIR].reshape(1, -1)
    raised = False
    try:
        torch.multinomial(row, 2048)
    except RuntimeError:
        raised = True
    assert raised == (draws.CONTRACT[case] == "zero")
