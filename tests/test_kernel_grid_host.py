"""CPU checks of the GEMM / attention case table (tests/kernel_grid.py): the restated dispatch rule, and that the table
reaches every regime cell, K residue, round shape, M tail, group order and epilogue variant at both H100 SM counts."""
import pytest

from tests import kernel_grid as kg


def test_dispatch_rule_at_known_shapes():
    """The restated launch_one at shapes whose regime the engine relies on (DESIGN.md §2, §4)."""
    L = kg.GemmLaunch
    # C3 (ViT-B, 64 images, T = 1939): attn.qkv 970 x 18 tiles, K = 12 chunks
    assert L("STORE_H", 64 * 1939, 2304, 12).regime == "persistent"
    assert L("STORE_H", 64 * 1939, 2304, 12).stages == 4
    # C2 (ViT-S, one pair): attn.proj 31 x 3 tiles, K = 6 chunks: deep ring; mlp.fc1 31 x 12: shallow
    assert L("RESID_F", 3878, 384, 6).regime == "deep"
    assert L("STORE_H", 3878, 1536, 6).regime == "shallow"
    # 64-wide tiles when N % 128 != 0, and their ring depths
    assert L("STORE_H", 50001, 192, 5).bn == 64 and L("STORE_H", 50001, 192, 5).stages == 6
    # the one-tile-only epilogues never take the persistent kernel; EPI_DUAL through TMA stores is always shallow
    assert L("LN", 80000, 128, 4, groups=4).regime == "shallow"
    assert L("DUAL", 128, 128, 6, groups=1, out_tma=True).regime == "shallow"
    assert L("DUAL", 128, 128, 6, groups=1, out_tma=False).regime == "deep"
    # the cutovers
    assert L("STORE_F", 128 * 165, 128, 4).regime == "deep" and L("STORE_F", 128 * 166, 128, 4).regime == "shallow"
    assert L("STORE_F", 128, 128, 3).regime == "shallow"
    assert L("STORE_F", 128 * 1056, 128, 1).regime == "shallow" and L("STORE_F", 128 * 1057, 128, 1).regime == "persistent"
    assert L("STORE_F", 128 * 912, 128, 1, sms=114).regime == "shallow"
    assert L("STORE_F", 128 * 913, 128, 1, sms=114).regime == "persistent"


def test_tile_walk():
    """gemm_tile order: N-tiles fastest, then the groups when they share A, then the M-tiles; own-A groups outermost.
    tile_of inverts it, and the persistent round is t // grid."""
    for fast in (False, True):
        L = kg.GemmLaunch("STORE_F", 1000, 384, 2, groups=3, group_fast=fast)
        seen = set()
        for t in range(L.tiles):
            g, m0, n0 = L.tile(t)
            assert L.index(g, m0, n0) == t
            seen.add((g, m0, n0))
        assert len(seen) == L.tiles
        assert L.tile(1) == (0, 0, 128)
        assert L.tile(3) == ((1, 0, 0) if fast else (0, 128, 0))
    P = kg.GemmLaunch("STORE_F", 128 * 1188, 128, 2)
    assert P.grid == 132 and P.rounds == 9 and P.tile_of(128 * 1187, 5)["round"] == 8


@pytest.mark.parametrize("sms", kg.SM_COUNTS)
def test_table_reaches_every_requirement(sms):
    cases = kg.gemm_cases(sms)
    assert not kg.coverage_gaps(cases, sms), kg.coverage_gaps(cases, sms)
    for c in cases:
        assert c.launch.regime == c.want, (c.name, c.launch.describe())
        assert c.sms == sms
    assert len({c.name for c in cases}) == len(cases)


@pytest.mark.parametrize("sms", kg.SM_COUNTS)
def test_removing_any_requirement_is_noticed(sms):
    """Taking out the cases that meet one requirement leaves a table the coverage check rejects, naming it."""
    cases = kg.gemm_cases(sms)
    for name, pred in kg.requirements(sms).items():
        rest = [c for c in cases if not pred(c)]
        assert len(rest) < len(cases), name
        assert name in kg.coverage_gaps(rest, sms), name


@pytest.mark.parametrize("sms", kg.SM_COUNTS)
def test_every_mutation_tile_is_in_the_last_round(sms):
    """The planted tile mutations sit in the last round of each launch, and the previous-round tile is the one the same
    persistent CTA ran before it."""
    n_persistent = 0
    for c in kg.gemm_cases(sms):
        L = c.launch
        t, tp = L.mutation_tiles()
        assert t // L.grid == L.rounds - 1
        if L.regime == "persistent":
            n_persistent += 1
            assert tp is not None and tp % L.grid == t % L.grid and tp // L.grid == L.rounds - 2, c.name
    assert n_persistent >= 10


@pytest.mark.parametrize("sms", kg.SM_COUNTS)
def test_attention_table(sms):
    cases = kg.attention_cases(sms)
    assert {c.T for c in cases} == set(kg.ATTN_T)
    for T in kg.ATTN_T:
        grids = {c.grid for c in cases if c.T == T}
        assert {"fewer tiles than SMs", "partial last round"} <= grids, (T, grids)
    assert sum(c.grid == "one tile per SM" for c in cases) >= 8
    # the key-leak cases: an even image whose last key tile is partial, followed by a scaled neighbour
    leaks = [c for c in cases if c.leak]
    assert all(c.n_img >= 2 for c in leaks)
    assert sum(c.T % 128 != 0 for c in leaks) >= 10
    # the logit scale is swept at every query-tile count
    assert {c.scale for c in cases} == set(kg.ATTN_SCALES)
