"""A table of GEMM and attention launches chosen to reach every launch regime of the two kernels that do most of the
work, with the dispatch rule of gemm.cu restated in Python so that the table can prove what it reaches.

The production shapes reach the regimes only where they happen to fall.  At C3 every persistent BN = 128 GEMM has
k_chunks = 0 or 2 (mod 4), so the persistent ring's stage and phase, which carry on from tile to tile, never start a
tile at ring stage 1 or 3; the cutovers between the one-tile rings and the persistent grid are met only by accident.
The cases below are built from the device's SM count (132 on an H100 SXM, 114 on a PCIe card), and
`coverage_gaps` names every regime cell, K residue, round shape, M tail, group order and epilogue variant the table
fails to reach.  tests/test_kernel_grid_host.py asserts, at both SM counts, that nothing is missing and that taking
away the cases of any one requirement is noticed.  tests/test_gpu_kernel_grid.py runs the cases against fp64.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

MATCHER = ("LSE", "DUAL")
ONE_TILE_ONLY = ("DUAL", "LN")                         # gemm_tc.cuh persistent_epilogue() is false for these
REGIMES = ("persistent", "deep", "shallow")
# ring depths (gemm_tc.cuh ring_stages / deep_stages / shallow_stages), by BN
STAGES = {"persistent": {128: 4, 64: 6}, "deep": {128: 6, 64: 8}, "shallow": {128: 3, 64: 4}}
SM_COUNTS = (132, 114)                                 # H100 SXM, H100 PCIe


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


@dataclass(frozen=True)
class GemmLaunch:
    """One launch_gemm call as gemm.cu dispatches it: tile width, tile count, regime, ring depth and the tile walk."""
    epi: str
    M: int
    N: int
    k_chunks: int
    groups: int = 1
    group_fast: bool = False          # groups share A (a_row_group_off == a_col_group_off == 0): group between M and N
    out_tma: bool = False             # EPI_DUAL with an output pitch % 4 == 0
    sms: int = 132

    @property
    def bn(self) -> int:
        return 128 if (self.epi in MATCHER or self.epi == "LN" or self.N % 128 == 0) else 64

    @property
    def m_tiles(self) -> int:
        return cdiv(self.M, 128)

    @property
    def n_tiles(self) -> int:
        return cdiv(self.N, self.bn)

    @property
    def tiles(self) -> int:
        return self.m_tiles * self.n_tiles * self.groups

    @property
    def regime(self) -> str:
        """gemm.cu launch_one: EPI_DUAL through TMA stores always takes the shallow ring; otherwise at most 5/4 tiles
        per SM with more than 3 K chunks take the deep ring; more than 8 tiles per SM take the persistent kernel (not
        for the one-tile-only epilogues); everything else the shallow ring."""
        if self.epi == "DUAL" and self.out_tma:
            return "shallow"
        if self.tiles <= self.sms * 5 // 4 and self.k_chunks > 3:
            return "deep"
        if self.epi not in ONE_TILE_ONLY and self.tiles > 8 * self.sms:
            return "persistent"
        return "shallow"

    @property
    def stages(self) -> int:
        return STAGES[self.regime][self.bn]

    @property
    def grid(self) -> int:
        return min(self.tiles, self.sms) if self.regime == "persistent" else self.tiles

    @property
    def rounds(self) -> int:
        return cdiv(self.tiles, self.grid)

    def tile(self, t: int):
        """gemm_tc.cuh gemm_tile: linear tile index -> (group, m0, n0)."""
        n = t % self.n_tiles
        t //= self.n_tiles
        if self.group_fast:
            g, m = t % self.groups, t // self.groups
        else:
            m, g = t % self.m_tiles, t // self.m_tiles
        return g, m * 128, n * self.bn

    def index(self, g: int, m0: int, n0: int) -> int:
        mt, nt = m0 // 128, n0 // self.bn
        return ((mt * self.groups + g) if self.group_fast else (g * self.m_tiles + mt)) * self.n_tiles + nt

    def tile_of(self, m: int, n: int, g: int = 0) -> dict:
        """The tile that writes output (m, n) of group g and the round that runs it (elementwise.Where protocol)."""
        t = self.index(g, m // 128 * 128, n // self.bn * self.bn)
        return dict(tile=t, m_tile=m // 128, n_tile=n // self.bn, group=g, round=t // self.grid, regime=self.describe())

    def describe(self) -> str:
        return f"{self.regime} BN={self.bn} {self.stages}-stage ring, grid {self.grid} of {self.tiles} tiles"

    def mutation_tiles(self):
        """(t, t_prev): the last tile, which runs in the LAST round, and the tile the same CTA ran one round earlier
        (for the one-tile regimes, whose single round is the last, the tile before it); t_prev None if there is none."""
        t = self.tiles - 1
        tp = t - self.grid if self.regime == "persistent" else t - 1
        return t, (tp if tp >= 0 else None)


@dataclass
class GemmCase:
    """A GEMM launch of the grid: the operands' layout, the epilogue and the regime it must reach."""
    name: str
    epi: str
    M: int
    N: int
    k_chunks: int
    want: str                              # the regime the case is there for
    groups: int = 1
    group_fast: bool = False
    a_col_base: int = 0
    a_row_group_off: int = 0
    a_col_group_off: int = 0
    b_row_group_off: int = 0
    act: int = 0                           # 0 none, 1 GELU, 2 ReLU
    bias: bool = False
    extra: dict = field(default_factory=dict)
    sms: int = 132

    @property
    def launch(self) -> GemmLaunch:
        out_tma = self.epi == "DUAL" and self.extra.get("pitch", 1) % 4 == 0
        return GemmLaunch(self.epi, self.M, self.N, self.k_chunks, self.groups, self.group_fast, out_tma, self.sms)

    @property
    def K(self) -> int:
        return 64 * self.k_chunks


def _m(m_tiles: int, tail: int) -> int:
    """M with m_tiles M-tiles whose last one holds `tail` rows (1..128)."""
    return 128 * (m_tiles - 1) + tail


# STORE_H / STORE_F / RESID_F variants rotated over the regime grid: (epi, act, bias)
_LINEAR_VARIANTS = (("STORE_H", 1, True), ("STORE_H", 0, True), ("STORE_H", 2, False), ("RESID_F", 0, True),
                    ("STORE_H", 0, False), ("STORE_F", 0, False), ("STORE_H", 1, False), ("STORE_H", 2, True))


def gemm_cases(sms: int) -> list:
    s = sms
    deep_max, p8, p9 = s * 5 // 4, 8 * s, 9 * s
    cases = []

    def add(name, epi, M, N, k, want, **kw):
        c = GemmCase(name, epi, M, N, k, want, sms=s, **kw)
        assert c.launch.regime == want, (name, c.launch.describe(), want)
        cases.append(c)

    # ---- regime x BN x K residue grid: (N, m_tiles, tail, k) per cell ----
    grid = {
        ("persistent", 128): [(128, p8 + 1, 1, 1), (128, p9, 64, 2), (128, p9 - 1, 127, 3), (128, p8 + 1, 128, 4),
                              (256, cdiv(p8 + 1, 2), 64, 5)],
        ("persistent", 64): [(64, p9, 1, 1), (64, p9 - 1, 64, 2), (64, p8 + 1, 127, 3), (192, p9 // 3, 128, 4),
                             (64, p9, 64, 5), (64, p8 + 1, 1, 6), (320, cdiv(p8 + 1, 5), 127, 7)],
        ("deep", 128): [(128, deep_max, 64, 4), (256, deep_max // 2, 127, 5), (128, 1, 77, 6), (384, 9, 1, 7),
                        (128, 40, 128, 8), (128, 3, 100, 9), (128, 1, 77, 4)],
        ("deep", 64): [(64, deep_max, 1, 4), (64, 1, 77, 5), (192, 7, 64, 6), (320, 3, 127, 7), (64, 60, 128, 8),
                       (192, 20, 3, 9), (64, 2, 64, 10), (320, 1, 127, 11)],
        ("shallow", 128): [(128, 1, 77, 1), (256, 5, 64, 2), (128, 1, 77, 3), (128, deep_max + 1, 127, 5),
                           (128, p8, 1, 6), (384, 150, 128, 7)],
        ("shallow", 64): [(64, 1, 30, 1), (192, 9, 127, 2), (64, 4, 64, 3), (64, deep_max + 1, 1, 4), (64, p8, 128, 8),
                          (320, 40, 64, 13)],
    }
    i = 0
    for (regime, bn), rows in grid.items():
        for N, mt, tail, k in rows:
            epi, act, bias = _LINEAR_VARIANTS[i % len(_LINEAR_VARIANTS)]
            i += 1
            add(f"{regime}_bn{bn}_k{k}_m{_m(mt, tail)}_n{N}_{epi.lower()}", epi, _m(mt, tail), N, k, regime, act=act, bias=bias or epi == "RESID_F")

    # ---- both group orders, non-zero a_col_base / a_row_group_off / b_row_group_off ----
    add("groups_shared_a_persistent", "STORE_F", _m(3 * s, 64), 128, 2, "persistent", groups=3, group_fast=True,
        a_col_base=64, b_row_group_off=160)
    add("groups_own_a_persistent", "STORE_H", _m(3 * s - 1, 100), 64, 3, "persistent", groups=3, a_col_base=64,
        a_row_group_off=_m(3 * s - 1, 100) + 40, a_col_group_off=64, b_row_group_off=128, act=1, bias=True)
    add("groups_shared_a_deep", "STORE_H", _m(9, 20), 128, 5, "deep", groups=4, group_fast=True, a_col_base=128,
        b_row_group_off=192, act=2, bias=True)
    add("groups_own_a_shallow", "STORE_F", _m(70, 90), 192, 2, "shallow", groups=2, a_col_base=64,
        a_row_group_off=_m(70, 90) + 8, b_row_group_off=256)

    # ---- EPI_PATCH: tok_per_img not a multiple of 128, so an image boundary (and the cls row it skips) is inside a tile
    add("patch_deep", "PATCH", 7 * 200, 384, 10, "deep", extra=dict(tok_per_img=200))
    n_img = cdiv((p8 + 1) * 128, 1000) + 1
    add("patch_persistent", "PATCH", n_img * 1000, 128, 10, "persistent", extra=dict(tok_per_img=1000))

    # ---- EPI_CONV: 3x3 taps as shifted rows over zero-padded NHWC grids, 4 groups with their own input columns ----
    # no pad mask: the first and last rows' taps reach rows before the first and after the last image (zero fill)
    add("conv_edges_bn128", "CONV", 2 * 12 * 10, 128, 9, "deep", extra=dict(n_img=2, h2=12, w2=10, cin=64, G=1, pad=False))
    add("conv_edges_bn64", "CONV", 3 * 11 * 9, 64, 18, "deep", extra=dict(n_img=3, h2=11, w2=9, cin=128, G=1, pad=False))
    # pad ring zeroed, fp16 shortcut, PE on the groups of each mask, fp32 and fp16 outputs together
    per = 40 * 53
    n_img = cdiv((2 * s + 1) * 128, per) + 1
    add("conv_pe_kp_persistent", "CONV", n_img * per, 128, 18, "persistent", groups=4, a_col_group_off=128,
        b_row_group_off=128, act=2, bias=True, extra=dict(n_img=n_img, h2=40, w2=53, cin=128, G=4, pad=True, mask=0x7))
    add("conv_pe_dsc_shallow", "CONV", 3 * per, 128, 18, "shallow", groups=4, a_col_group_off=128, b_row_group_off=128,
        act=2, bias=True, extra=dict(n_img=3, h2=40, w2=53, cin=128, G=4, pad=True, mask=0x8))
    add("conv_pe_all_deep_small", "CONV", 1 * 10 * 12, 128, 18, "deep", groups=4, a_col_group_off=128,
        b_row_group_off=128, act=2, bias=True, extra=dict(n_img=1, h2=10, w2=12, cin=128, G=4, pad=True, mask=0xF))
    add("conv_no_pe_bn64", "CONV", 16 * 22 * 17, 64, 9, "shallow", groups=4, a_col_group_off=64, b_row_group_off=64,
        act=2, bias=True, extra=dict(n_img=16, h2=22, w2=17, cin=64, G=4, pad=True, mask=0x0))

    # ---- EPI_LN (N = 128), grouped, with the fp32 residual and the pad mask ----
    add("ln_own_a_deep", "LN", 2 * 20 * 22, 128, 4, "deep", groups=4, a_col_group_off=256, b_row_group_off=128,
        extra=dict(n_img=2, h2=20, w2=22))
    add("ln_own_a_shallow", "LN", 8 * 40 * 53, 128, 4, "shallow", groups=4, a_col_group_off=256, b_row_group_off=128,
        extra=dict(n_img=8, h2=40, w2=53))
    add("ln_shared_a_shallow", "LN", 3 * 30 * 31, 128, 3, "shallow", groups=2, group_fast=True, a_col_base=64,
        b_row_group_off=128, extra=dict(n_img=3, h2=30, w2=31))

    # ---- the matcher: EPI_LSE -> mk_op_matcher_reduce -> EPI_DUAL ----
    for n, B, confs in ((2, 3, ((0.0, False, False), (1.001, True, True))),
                        (127, 2, ((1.001, False, False), (0.0, True, True))),
                        (128, 2, ((0.0, True, False), (1.001, False, True))),
                        (129, 2, ((1.001, True, False), (0.0, False, True))),
                        (1938, 5, ((0.0, False, False), (1.001, True, True)))):
        for bound, tma, lean in confs:
            pitch = cdiv(n, 32) * 32 if tma else (n if n % 4 else n + 2)
            tag = f"n{n}_{'bounded' if bound else 'maxima'}_{'tma' if tma else 'stg'}{'_lean' if lean else ''}"
            ex = dict(B=B, lse_bound=bound, pitch=pitch, lean=lean)
            lse = GemmLaunch("LSE", n, n, 6, B, sms=s)
            add(f"lse_{tag}", "LSE", n, n, 6, lse.regime, groups=B, a_row_group_off=n, b_row_group_off=n, extra=ex)
            dual = GemmLaunch("DUAL", n, n, 6, B, out_tma=tma, sms=s)
            add(f"dual_{tag}", "DUAL", n, n, 6, dual.regime, groups=B, a_row_group_off=n, b_row_group_off=n, extra=ex)
    return cases


# ---------------------------------------------------------------------------------------------------------------
# what the table must reach
# ---------------------------------------------------------------------------------------------------------------
def requirements(sms: int) -> dict:
    """name -> predicate over a GemmCase.  Every name needs at least one case."""
    s = sms
    req = {}
    L = lambda c: c.launch                                                     # noqa: E731
    for regime in REGIMES:
        for bn in (64, 128):
            req[f"{regime} BN={bn}"] = lambda c, r=regime, b=bn: L(c).regime == r and L(c).bn == b
            st = STAGES[regime][bn]
            for res in range(st):
                req[f"{regime} BN={bn} k_chunks = {res} mod {st}"] = (
                    lambda c, r=regime, b=bn, st=st, res=res: L(c).regime == r and L(c).bn == b and L(c).k_chunks % st == res)
    for regime in ("persistent", "shallow"):
        for bn in (64, 128):
            for k in (1, 2, 3):
                req[f"{regime} BN={bn} k_chunks = {k}"] = (
                    lambda c, r=regime, b=bn, k=k: L(c).regime == r and L(c).bn == b and L(c).k_chunks == k)
    for tiles, what in ((8 * s + 1, "8 SMs + 1"), (9 * s, "9 SMs"), (9 * s - 1, "9 SMs - 1")):
        req[f"persistent grid of {what} tiles"] = lambda c, t=tiles: L(c).regime == "persistent" and L(c).tiles == t
    # the cutovers of launch_one, from both sides
    req["deep at 5/4 tiles per SM"] = lambda c: L(c).regime == "deep" and L(c).tiles == s * 5 // 4
    req["shallow at 5/4 tiles per SM + 1, k_chunks > 3"] = (
        lambda c: L(c).regime == "shallow" and L(c).tiles == s * 5 // 4 + 1 and L(c).k_chunks > 3)
    req["shallow at 8 tiles per SM"] = lambda c: L(c).regime == "shallow" and L(c).tiles == 8 * s
    req["shallow with one tile and k_chunks = 3"] = lambda c: L(c).regime == "shallow" and L(c).tiles == 1 and L(c).k_chunks == 3
    req["deep with one tile and k_chunks = 4"] = lambda c: L(c).regime == "deep" and L(c).tiles == 1 and L(c).k_chunks == 4
    for tail in (0, 1, 64, 127):
        req[f"M = {tail} mod 128"] = lambda c, t=tail: c.epi not in MATCHER and c.M % 128 == t and c.M > 128
    req["M < 128"] = lambda c: c.epi not in MATCHER and c.M < 128
    req["groups sharing A (group-fast order), a_col_base, b_row_group_off"] = (
        lambda c: c.groups > 1 and c.group_fast and c.a_col_base > 0 and c.b_row_group_off > 0)
    req["groups with their own A, a_col_base, a_row_group_off, b_row_group_off"] = (
        lambda c: c.groups > 1 and not c.group_fast and c.a_col_base > 0 and c.a_row_group_off > 0 and c.b_row_group_off > 0)
    for fast in (True, False):
        req[f"persistent groups, {'group-fast' if fast else 'own A'}"] = (
            lambda c, f=fast: c.groups > 1 and c.group_fast == f and c.epi not in MATCHER and L(c).regime == "persistent")
    # epilogue variants
    for act in (0, 1, 2):
        for bias in (False, True):
            req[f"STORE_H act {act} bias {bias}"] = lambda c, a=act, b=bias: c.epi == "STORE_H" and c.act == a and c.bias == b
    for epi in ("STORE_F", "RESID_F", "PATCH", "LN"):
        req[f"{epi}"] = lambda c, e=epi: c.epi == e
    req["PATCH image boundary inside a tile"] = lambda c: c.epi == "PATCH" and c.extra["tok_per_img"] % 128 != 0
    req["CONV without pad mask (taps off both ends)"] = lambda c: c.epi == "CONV" and not c.extra["pad"]
    for mask in (0x0, 0x7, 0x8, 0xF):
        req[f"CONV pad ring, shortcut, aux_group_mask {mask:#x}"] = (
            lambda c, m=mask: c.epi == "CONV" and c.extra["pad"] and c.extra.get("mask") == m)
    for n in (2, 127, 128, 129, 1938):
        req[f"matcher n_valid {n}"] = lambda c, n=n: c.epi == "DUAL" and c.M == n
    for bound in (False, True):
        for tma in (False, True):
            req[f"matcher lse_bound {bound} tma {tma}"] = (
                lambda c, b=bound, t=tma: c.epi == "DUAL" and bool(c.extra["lse_bound"]) == b and L(c).out_tma == t)
        req[f"matcher lean, tma {bound}"] = lambda c, t=bound: c.epi == "DUAL" and c.extra["lean"] and L(c).out_tma == t
    req["LSE on the persistent grid"] = lambda c: c.epi == "LSE" and L(c).regime == "persistent"
    return req


def coverage_gaps(cases, sms: int) -> list:
    return [name for name, pred in requirements(sms).items() if not any(pred(c) for c in cases)]


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
ATTN_T = (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 383, 384, 385, 1939)
ATTN_BQ, ATTN_BK = 192, 128
ATTN_SCALES = (1.5, 6.0, 3.0)


@dataclass(frozen=True)
class AttnCase:
    name: str
    T: int
    n_img: int
    heads: int
    scale: float              # std of the fp16 q, k, v entries
    leak: bool                # the K of every odd image scaled x50 (the last key tile of image 2i reads image 2i+1)
    sms: int = 132

    @property
    def q_tiles(self) -> int:
        return cdiv(self.T, ATTN_BQ)

    @property
    def tiles(self) -> int:
        return self.q_tiles * self.heads * self.n_img

    @property
    def grid(self) -> str:
        if self.tiles < self.sms:
            return "fewer tiles than SMs"
        if self.tiles == self.sms:
            return "one tile per SM"
        return "partial last round" if self.tiles % self.sms else "full rounds"


def _exact(q: int, sms: int) -> Optional[tuple]:
    """(heads, n_img) with q * heads * n_img == sms, heads <= 16 as large as possible."""
    if sms % q:
        return None
    r = sms // q
    for h in range(min(16, r), 0, -1):
        if r % h == 0:
            return h, r // h
    return None


def attention_cases(sms: int) -> list:
    out = []
    for i, T in enumerate(ATTN_T):
        q = cdiv(T, ATTN_BQ)
        sc = ATTN_SCALES[i % len(ATTN_SCALES)]
        out.append(AttnCase(f"T{T}_fewer", T, 2, 2, sc, False, sms))
        ex = _exact(q, sms)
        if ex is not None:
            out.append(AttnCase(f"T{T}_exact", T, ex[1], ex[0], ATTN_SCALES[(i + 1) % len(ATTN_SCALES)], False, sms))
        heads = 6
        n_img = max(2, cdiv(sms + 1, q * heads))
        while (q * heads * n_img) % sms == 0:
            n_img += 1
        out.append(AttnCase(f"T{T}_partial_leak", T, n_img, heads, 1.5, True, sms))
    return out
