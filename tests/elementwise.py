"""Element-wise checks of kernel outputs against fp64 references, with error bounds derived from the arithmetic.

`check` asserts |got - ref| <= bound for EVERY element (not a Frobenius norm over the tensor, which hides a wrong tile:
one 32-column chunk of one row left at zero in a 50,000 x 192 output moves the relative Frobenius error by ~2e-3).  On
failure it names the stage, the number of failing elements and the worst one, mapped back to (image, position, group,
column) and, for GEMM outputs, to its tile in `gemm_tile` order and the persistent round that ran it.

Every check also runs against `Mutation`s of its reference -- the bug a tiling change would introduce (a K chunk dropped
from one tile, a conv tap read one padded row off, a token of the neighbouring image, the PE row of the neighbouring
position, a 32-column chunk of the next row, hi and lo swapped in the split descriptor) -- and asserts that the bound
rejects each of them.  A bound loose enough to let one through fails the test instead of passing silently.

Bounds (u32 = 2^-24, the fp32 unit roundoff; u16 = 2^-11, fp16's).  None of them is fitted to observed errors: where a
bound turned out too tight for a correct kernel, the formula was re-derived (see the notes at each function).

* GEMM family, fp16 operands, fp32 accumulation over K products:
      |acc - A64 B64^T| <= K * 2^-23 * (|A| |B|^T)
  (2^-23 rather than the round-to-nearest 2^-24: the tensor-core adders may truncate instead of rounding).  Every fp32
  epilogue operation adds at most u32 of its result; `epilogue_terms` charges 4 u32 of the sum of the magnitudes of
  the terms (bias, LayerScale product, residual, PE).  The exact-erf GELU (Abramowitz-Stegun 7.1.26 with MUFU rcp/ex2)
  adds 5e-7 * (1 + |x|), and its slope (<= 1.13) scales the error of its argument; ReLU is 1-Lipschitz.
  Output rounding: 2^-11 |ref| + 2^-24 for fp16 (2^-24 covers the subnormal range), 2^-24 |ref| for fp32.
* LayerNorm of a row x_1..x_D whose elements carry errors <= e_i (E = max e_i), computed in fp32:
      d_i = x_i - mu,  sigma^2 = mean(d^2),  r = (sigma^2 + eps)^-1/2
      |d mu|      <= E + D u32 mean|x|                          (= E_mu)
      |d d_i|     <= e_i + E_mu + u32 |d_i|
      |d sigma^2| <= 2 sigma (E + E_mu) + (D + 2) u32 sigma^2
      |d r| / r   <= |d sigma^2| / (2 (sigma^2 + eps)) + 2^-22        (rsqrtf: 2 ulp)
      |d y_i|     <= |gamma_i| r (|d d_i| + |d_i| |d r|/r) + 3 u32 (|d_i r gamma_i| + |beta_i|)
  then output rounding.
* Attention (fp16 Q, K, V; S and P.V accumulated in fp32; P rounded to fp16 once, the row sum l taken from the
  unrounded P): with eps_s = 64 * 2^-23 * (|q| |k|^T) / 8 + 2^-23 |s| the error of a logit and
  eps = max_j eps_s + 2^-21 (ex2.approx),
      |d o| <= (2^-11 + 2 eps + (T + 64) 2^-23) sum_j p_j |v_j|      (P rounding, logits, P.V accumulation)
             + 2^-25 sum_j |v_j| / l                                (P below fp16's normal range: absolute 2^-25)
             + (eps + T u32) |o| + 2^-11 |o| + 2^-24                 (row sum, output rounding)
  with p the normalised fp64 softmax and l = sum_j exp(s_j - max s).
* fp32 reductions (linear attention, head outputs, descriptor normalisation, matcher log-sum-exp):
      |sum - exact| <= n u32 sum |terms|   for n terms in any order,
  plus a few u32 per elementary operation and 2 ulp (2^-22 relative) per expf / sqrtf / ex2.approx / log2f.
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import dataclass, field
from typing import Callable, Optional, Sequence

import torch

U32 = 2.0 ** -24
U16 = 2.0 ** -11
GELU_SLOPE = 1.13                    # max |GELU'(x)| = 1.1289 at x = +-sqrt(2)
GELU_APPROX = 5e-7                   # A-S 7.1.26 (1.5e-7 in erf) * |x|/2 plus the MUFU rcp / ex2 ulps
SM_COUNT_H100 = 132


# ---------------------------------------------------------------------------------------------------------------
# bounds
# ---------------------------------------------------------------------------------------------------------------
def gemm_acc_bound(K: int, abs_prod: torch.Tensor) -> torch.Tensor:
    """fp32 accumulation of K fp16 x fp16 products: K 2^-23 (|A| |B|^T)."""
    return K * 2.0 ** -23 * abs_prod


def epilogue_terms(*terms) -> torch.Tensor:
    """4 u32 times the sum of the magnitudes of the fp32 epilogue terms (accumulator, bias, residual, PE, ...)."""
    tot = None
    for t in terms:
        if t is None:
            continue
        a = t.abs() if torch.is_tensor(t) else abs(t)
        tot = a if tot is None else tot + a
    return 4 * U32 * tot


def out_rounding(ref: torch.Tensor, fp16: bool) -> torch.Tensor:
    return U16 * ref.abs() + U32 if fp16 else U32 * ref.abs()


def gelu64(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_bound(x: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """Error of GELU(x~) against GELU(x) when |x~ - x| <= e."""
    return GELU_SLOPE * e + GELU_APPROX * (1.0 + x.abs() + e)


def ln_bound(x: torch.Tensor, e: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float):
    """(fp64 LayerNorm of the rows of x, bound on the fp32 kernel's error) for rows whose elements carry errors <= e
    (same shape as x, or a scalar).  See the module docstring for the derivation."""
    D = x.shape[-1]
    e = torch.as_tensor(e, dtype=torch.float64, device=x.device).expand_as(x)
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    var = (d * d).mean(-1, keepdim=True)
    r = torch.rsqrt(var + eps)
    y = d * r * gamma + beta
    E = e.amax(-1, keepdim=True)
    E_mu = E + D * U32 * x.abs().mean(-1, keepdim=True)
    dd = e + E_mu + U32 * d.abs()
    sigma = var.sqrt()
    dvar = 2 * sigma * (E + E_mu) + (D + 2) * U32 * var
    dr = dvar / (2 * (var + eps)) + 2.0 ** -22
    b = gamma.abs() * r * (dd + d.abs() * dr) + 3 * U32 * ((d * r * gamma).abs() + beta.abs())
    return y, b


# ---------------------------------------------------------------------------------------------------------------
# coordinates of an element: where it lives and which GEMM tile / persistent round produced it
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class Rows:
    """How a row index maps to an image: `padded` rows of (h2 x w2) grids, `tokens` rows of T tokens (cls first),
    `patches` rows of N patch tokens, or `flat`."""
    kind: str = "flat"
    per_img: int = 1
    w2: int = 1

    def describe(self, m: int) -> str:
        if self.kind == "flat":
            return f"row {m}"
        img, p = divmod(int(m), self.per_img)
        if self.kind == "padded":
            y, x = divmod(p, self.w2)
            return f"image {img}, padded position {p} (y {y}, x {x})"
        if self.kind == "tokens":
            return f"image {img}, token {p}" + (" (cls)" if p == 0 else "")
        return f"image {img}, patch {p}"


@dataclass
class GemmTiles:
    """The tile walk of one GEMM launch (gemm_tc.cuh gemm_tile): N-tiles fastest, then the groups if they share A
    (group_fast), then the M-tiles; groups with their own A outermost.  Grids of more than 8 tiles per SM run
    persistent CTAs (one per SM) striding through the tiles: tile t runs in round t // grid."""
    M: int
    N: int
    groups: int = 1
    group_fast: bool = False
    sms: int = SM_COUNT_H100

    @property
    def bn(self) -> int:
        return 128 if self.N % 128 == 0 else 64

    @property
    def tiles(self) -> int:
        return -(-self.M // 128) * (self.N // self.bn) * self.groups

    @property
    def persistent(self) -> bool:
        return self.tiles > 8 * self.sms

    def tile_of(self, m: int, n: int, g: int = 0):
        mt, nt, n_tiles, m_tiles = m // 128, n // self.bn, self.N // self.bn, -(-self.M // 128)
        t = ((mt * self.groups + g) if self.group_fast else (g * m_tiles + mt)) * n_tiles + nt
        grid = min(self.tiles, self.sms) if self.persistent else self.tiles
        return dict(tile=t, m_tile=mt, n_tile=nt, group=g, round=t // grid,
                    regime="persistent" if self.persistent else "one tile per CTA")


@dataclass
class Where:
    """Maps an index of the checked tensor to words.  `coords(idx)` -> (row, group, column) of the GEMM output (or
    None to print the raw index); `rows` names the row; `tiles` adds the tile."""
    coords: Optional[Callable] = None
    rows: Rows = field(default_factory=Rows)
    tiles: Optional[GemmTiles] = None
    row_offset: int = 0

    def describe(self, idx) -> str:
        if self.coords is None:
            return f"index {tuple(idx)}"
        m, g, n = self.coords(idx)
        m += self.row_offset
        s = f"{self.rows.describe(m)}, group {g}, column {n} (index {tuple(idx)})"
        if self.tiles is not None:
            t = self.tiles.tile_of(m, n, g)
            s += (f"; GEMM tile {t['tile']} (M-tile {t['m_tile']}, N-tile {t['n_tile']}, group {t['group']}), "
                  f"{t['regime']} round {t['round']}")
        return s


def matrix_where(rows: Optional[Rows] = None, tiles: Optional[GemmTiles] = None, group_width: Optional[int] = None,
                 row_offset: int = 0) -> Where:
    """A [rows, columns] output; with group_width the columns are [group][group_width]."""
    def coords(idx):
        m, c = int(idx[0]), int(idx[-1])
        if group_width:
            return m, c // group_width, c % group_width
        return m, 0, c
    return Where(coords, rows or Rows(), tiles, row_offset)


# ---------------------------------------------------------------------------------------------------------------
# mutations and the check itself
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class Mutation:
    """ref with ref[idx] replaced by `values` (the reference a specific bug would produce)."""
    label: str
    idx: tuple
    values: torch.Tensor


def row_chunk_swap(ref: torch.Tensor, row: int, col0: int, width: int = 32) -> Mutation:
    """One row's 32-column chunk replaced by the next row's (a mis-addressed epilogue row)."""
    return Mutation(f"row {row} columns {col0}..{col0 + width - 1} taken from row {row + 1}",
                    (slice(row, row + 1), slice(col0, col0 + width)), ref[row + 1:row + 2, col0:col0 + width].clone())


_METRICS: dict = {}


def record(stage: str, geometry: str, ratio: float) -> None:
    """max(err / bound) per stage and geometry -> the JSON file named by $MICKEY_STAGE_METRICS (merged with what is
    there, so that several runs of the suite accumulate)."""
    path = os.environ.get("MICKEY_STAGE_METRICS")
    _METRICS.setdefault(geometry, {})[stage] = float(ratio)
    if not path:
        return
    old = {}
    if os.path.exists(path):
        try:
            with open(path) as f:
                old = json.load(f)
        except (OSError, ValueError):
            old = {}
    for g, d in _METRICS.items():
        old.setdefault(g, {}).update(d)
    with open(path, "w") as f:
        json.dump(old, f, indent=1, sort_keys=True)


def check(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, where: Optional[Where] = None,
          mutations: Sequence[Mutation] = ()) -> float:
    """Assert |got - ref| <= bound element-wise (ref fp64); assert that every mutation of ref is rejected.
    Returns max(err / bound)."""
    assert got.shape == ref.shape, (name, tuple(got.shape), tuple(ref.shape))
    where = where or Where()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(ref)
    assert bool((bound > 0).all()), f"{name}: bounds must be positive"
    g = got.double()
    err = (g - ref).abs()
    ratio = err / bound
    ratio = torch.where(torch.isfinite(g), ratio, torch.full_like(ratio, float("inf")))
    worst = float(ratio.max())
    if not worst <= 1.0:
        n_bad = int((ratio > 1.0).sum())
        flat = int(ratio.argmax())
        idx = torch.unravel_index(torch.tensor(flat), ratio.shape)
        idx = tuple(int(i) for i in idx)
        raise AssertionError(
            f"{name}: {n_bad} of {ratio.numel()} elements outside the bound; worst err/bound {worst:.3g} at "
            f"{where.describe(idx)}: got {float(g[idx]):.9g}, ref {float(ref[idx]):.9g}, bound {float(bound[idx]):.3g}")
    for mu in mutations:
        gm = g[mu.idx]
        rejected = bool(((gm - mu.values.double()).abs() > bound[mu.idx]).any())
        assert rejected, f"{name}: the bound does not reject the mutation '{mu.label}'"
    return worst


def check_exact(name: str, got: torch.Tensor, ref: torch.Tensor, where: Optional[Where] = None,
                mutations: Sequence[Mutation] = ()) -> float:
    """Bit equality; each mutation must differ from got somewhere.  Returns 0.0 (err / bound is 0 by definition)."""
    assert got.shape == ref.shape and got.dtype == ref.dtype, (name, got.shape, ref.shape, got.dtype, ref.dtype)
    where = where or Where()
    same = (got == ref) | (torch.isnan(got) & torch.isnan(ref)) if got.is_floating_point() else (got == ref)
    if not bool(same.all()):
        bad = ~same
        flat = int(bad.reshape(-1).nonzero()[0])
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), got.shape))
        raise AssertionError(f"{name}: {int(bad.sum())} of {got.numel()} elements differ; first at {where.describe(idx)}: "
                             f"got {got[idx].item()!r}, ref {ref[idx].item()!r}")
    for mu in mutations:
        assert not torch.equal(got[mu.idx], mu.values.to(got.dtype)), f"{name}: the mutation '{mu.label}' is not rejected"
    return 0.0


def attention_ref_bound(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float = 0.125):
    """fp64 softmax(q k^T * scale) v over [..., T, 64] operands holding the kernel's exact fp16 values, and the bound
    of the module docstring."""
    T = k.shape[-2]
    s = (q @ k.transpose(-1, -2)) * scale
    eps = (64 * 2.0 ** -23 * scale * (q.abs() @ k.abs().transpose(-1, -2)) + 2.0 ** -23 * s.abs()).amax(-1, keepdim=True)
    eps = eps + 2.0 ** -21
    e = torch.exp(s - s.amax(-1, keepdim=True))
    del s
    l = e.sum(-1, keepdim=True)
    p = e / l
    del e
    o = p @ v
    pv = p @ v.abs()
    del p
    bound = ((U16 + 2 * eps + (T + 64) * 2.0 ** -23) * pv + 2.0 ** -25 * v.abs().sum(-2, keepdim=True) / l
             + (eps + T * U32 + U16) * o.abs() + U32)
    return o, bound


def split_hi_lo(d: torch.Tensor):
    """fp32 descriptor -> (hi, lo) fp16 with hi = rn(d), lo = rn(d - hi) (the matcher's split operand)."""
    hi = d.half()
    return hi, (d - hi.float()).half()
