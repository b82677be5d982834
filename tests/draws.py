"""Plain-torch restatements of the solver's two random draws (ransac.cu), on the CPU or the GPU.

Outer draw.  For every stream s of pair b the sampler runs the exponential race "the n_s largest p_e / Exp(1)" over the
cells e = i * N + j of final_scores (ATen's multinomial without replacement is top-k of p / Exp(1)).  Its uniform is
48 bits wide:

    prefix16 = half (j & 1) of word (j >> 1) of Philox(seed)(e, (e >> 32) ^ 0x5bd1e995, s >> 3, b),  j = s & 7
    low32    = word 0 of Philox(seed)(e, (e >> 32) ^ 0x2545F491, s, b)
    u        = (prefix16 + (low32 + 1/2) 2^-32) 2^-16,     key = p / -log1p(-u)

`outer_keys` evaluates the keys in fp64; `reference_draw` is the n_s largest of them in ascending cell order.

Key error of the kernel.  The kernel forms u in fp32 and E = -log1p(-u) as a 4-term series for u < 0.01 (truncation
u^5 / 5 < 2e-11 relative) or as -__logf(1 - u) above.  __logf has an absolute error of 2^-21.41 on [0.5, 2]; 1 - u
is exact there (Sterbenz) and E >= -log(0.99) = 0.01005, so the relative error of E is at most
2^-21.41 / 0.01005 = 3.6e-5.  The fp32 rounding of u (2^-25 absolute near u = 1) adds 2^-25 / ((1 - u) E), which is
below 1e-5 for E < 8 and grows beyond that; a cell with E > 8 can only sit at the boundary key k* if p = E k* > 8 k*,
and such a cell is drawn unless its E is that large (probability e^-8 = 3e-4 per cell, and then it lies far below k*
unless p is still larger).  __fdividef adds 2 ulp (1.2e-7).  So the kernel's key is within about 4e-5 of the fp64 key,
and its draw may differ from the fp64 draw only in cells whose fp64 key lies within 1e-4 of k*, the fp64 n_s-th
largest key: `band_check`.

Inner draw.  Each hypothesis h of set s_in of pair b draws 3 of the set's n_s entries without replacement with
probability proportional to the weights w_i = final_scores at the set's cells, by successive sampling on the cdf.  The
kernel is deterministic, so `inner_cdf` and `inner_draw` restate it bit for bit in fp32: the cdf in the kernel's
summation order, the uniforms of Philox(seed ^ 0x9E3779B97F4A7C15)(h, s_in, b, 0x3c6ef372), the removal of the drawn
mass, the skip over drawn entries, the clamp below W and the guard.  `law3` is the closed-form law of successive
sampling.

The training loss (loss.cu, loss_hyp_kernel) draws C of its S set entries the same way, generalised: `loss_inner_cdf`
is the cdf of its thread layout (S a multiple of 32, thread t owns entries t * ceil(S / 256) + j < S), and
`loss_inner_draw` its C draws, with key seed ^ 0x9E3779B97F4A7C15, counters (h, s_in, b, 0xA54FF53A + k / 4) and the four
words of one Philox call used by draws 4 (k / 4) .. 4 (k / 4) + 3.
"""
import itertools
import math

import torch

MASK32 = 0xFFFFFFFF
PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85
TAG_PREFIX, TAG_LOW = 0x5BD1E995, 0x2545F491
INNER_SEED_XOR, INNER_TAG = 0x9E3779B97F4A7C15, 0x3C6EF372
LOSS_INNER_TAG = 0xA54FF53A                      # loss.cu: 4th Philox counter of the loss's inner draw, + k / 4
HYP_THREADS = 256                                # ransac_solve_kernel's block: the cdf is scanned across these threads
LOSS_THREADS = 256                               # loss_hyp_kernel's block
BAND = 1e-4                                      # relative key band around k* (module docstring)
F32_ONE_MINUS_ULP = 1.0 - 2.0 ** -24             # 0.99999994f


# ---------------------------------------------------------------------------------------------------------------
# Philox4x32-7 on int64 tensors
# ---------------------------------------------------------------------------------------------------------------
def _mulhilo(m: int, x: torch.Tensor):
    """(hi, lo) 32-bit words of m * x for a 32-bit constant m and x in [0, 2^32): x is split into 16-bit limbs so that
    every int64 product stays below 2^48."""
    p_lo, p_hi = (x & 0xFFFF) * m, (x >> 16) * m
    s = p_lo + ((p_hi & 0xFFFF) << 16)
    return (p_hi >> 16) + (s >> 32), s & MASK32


def philox(c0, c1, c2, c3, seed: int, device=None):
    """Philox4x32-7 of ransac.cu (struct Philox): counters are int64 tensors or ints holding 32-bit values; returns
    the four output words as int64 tensors of the broadcast shape."""
    dev = next((c.device for c in (c0, c1, c2, c3) if torch.is_tensor(c)), device)
    ts = [torch.as_tensor(c, dtype=torch.int64, device=dev) & MASK32 for c in (c0, c1, c2, c3)]
    c0, c1, c2, c3 = torch.broadcast_tensors(*ts)
    k0, k1 = seed & MASK32, (seed >> 32) & MASK32
    for _ in range(7):
        hi0, lo0 = _mulhilo(PHILOX_M0, c0)
        hi1, lo1 = _mulhilo(PHILOX_M1, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + PHILOX_W0) & MASK32, (k1 + PHILOX_W1) & MASK32
    return c0, c1, c2, c3


# ---------------------------------------------------------------------------------------------------------------
# outer draw
# ---------------------------------------------------------------------------------------------------------------
def outer_keys(p: torch.Tensor, seed: int, b: int, streams, chunk: int = 1 << 22):
    """Yield (s, key) for each stream s: key fp64 [cells] = p / -log1p(-u) on the cells with p > 0, else 0.
    p: fp64 [cells], logical (row-major, unpadded) cell order.  The prefix words of a group of 8 streams come from one
    Philox call, as in the kernel; the work is chunked by cells so that 3.76 M cells fit in memory."""
    cells = p.numel()
    dev = p.device
    streams = list(streams)
    groups = sorted({s >> 3 for s in streams})
    keys = {s: torch.zeros(cells, dtype=torch.float64, device=dev) for s in streams}
    for c0 in range(0, cells, chunk):
        e = torch.arange(c0, min(cells, c0 + chunk), dtype=torch.int64, device=dev)
        pe = p[c0:c0 + e.numel()]
        pos = pe > 0
        for g in groups:
            words = philox(e & MASK32, (e >> 32) ^ TAG_PREFIX, g, b, seed)
            for s in (s for s in streams if s >> 3 == g):
                j = s & 7
                prefix = (words[j >> 1] >> (16 * (j & 1))) & 0xFFFF
                low = philox(e & MASK32, (e >> 32) ^ TAG_LOW, s, b, seed)[0]
                u = (prefix.double() + (low.double() + 0.5) * 2.0 ** -32) * 2.0 ** -16
                keys[s][c0:c0 + e.numel()] = torch.where(pos, pe / -torch.log1p(-u), torch.zeros_like(pe))
    for s in streams:
        yield s, keys[s]


def reference_draw(key: torch.Tensor, n_s: int) -> torch.Tensor:
    """The n_s largest keys, in ascending cell order (the kernel's canonical order of a draw)."""
    return torch.topk(key, n_s).indices.sort().values


def fill_draw(p: torch.Tensor, n_s: int) -> torch.Tensor:
    """The draw of a matrix with 0 < positive cells < n_s: every positive cell, then the lowest-index zero cells."""
    pos = (p > 0).nonzero()[:, 0]
    free = (p <= 0).nonzero()[:, 0][: n_s - pos.numel()]
    return torch.cat([pos, free]).sort().values


def band_check(got: torch.Tensor, key: torch.Tensor, n_s: int, band: float = BAND) -> dict:
    """Compare a kernel draw with the fp64 race.  Returns the counts; `ok` is True when the draw is n_s distinct
    in-range cells in ascending order and every cell in which it differs from the fp64 top n_s has |key / k* - 1| <=
    band (k* = the fp64 n_s-th largest key)."""
    got = got.to(key.device, torch.int64)
    cells = key.numel()
    shape_ok = got.numel() == n_s and bool((got >= 0).all()) and bool((got < cells).all()) and bool((got[1:] > got[:-1]).all())
    top = torch.topk(key, n_s)
    kstar = float(top.values[-1])
    in_ref = torch.zeros(cells, dtype=torch.bool, device=key.device)
    in_ref[top.indices] = True
    in_got = torch.zeros_like(in_ref)
    if shape_ok:
        in_got[got] = True
    rel = (key / kstar - 1.0).abs() if kstar > 0 else torch.full_like(key, float("inf"))
    diff = in_ref ^ in_got
    bad = diff & ~(rel <= band)
    return {"ok": shape_ok and kstar > 0 and int(bad.sum()) == 0, "n_diff": int(diff.sum()), "n_bad": int(bad.sum()),
            "n_band": int((rel <= band).sum()), "kstar": kstar}


# ---------------------------------------------------------------------------------------------------------------
# inner draw, bit-exact in fp32
# ---------------------------------------------------------------------------------------------------------------
def inner_cdf(w: torch.Tensor) -> torch.Tensor:
    """fp32 [S, n_s] weights -> the kernel's fp32 cdf [S, n_s] (ransac_solve_kernel, gather_set): thread t adds its
    n_s / 256 weights serially; a shfl_up warp scan of the thread totals; the exclusive base inc - run; then the totals
    of the preceding warps, one by one in warp order; cdf = thread-local running sum + base."""
    S, n = w.shape
    per = n // HYP_THREADS
    wv = w.float().reshape(S, HYP_THREADS, per)
    run = torch.zeros(S, HYP_THREADS, dtype=torch.float32, device=w.device)
    loc = torch.empty_like(wv)
    for j in range(per):
        run = run + wv[:, :, j]
        loc[:, :, j] = run
    return (loc + _scan_base(run)[:, :, None]).reshape(S, n)


def _scan_base(run: torch.Tensor) -> torch.Tensor:
    """The exclusive base of every thread's run total [S, threads]: a shfl_up warp scan, inc - run, then the totals of
    the preceding warps added one by one in warp order."""
    threads = run.shape[1]
    t = torch.arange(threads, device=run.device)
    lane, warp = t % 32, t // 32
    inc = run.clone()
    for o in (1, 2, 4, 8, 16):
        inc = torch.where(lane >= o, inc + torch.roll(inc, o, dims=1), inc)
    wtot = inc.reshape(run.shape[0], threads // 32, 32)[:, :, 31]
    base = inc - run
    for wi in range(threads // 32 - 1):
        base = torch.where(warp > wi, base + wtot[:, wi:wi + 1], base)
    return base


def loss_inner_cdf(w: torch.Tensor) -> torch.Tensor:
    """fp32 [R, S] weights -> loss_hyp_kernel's fp32 cdf [R, S] for any S that is a multiple of 32: with per =
    ceil(S / 256), thread t adds the weights of entries t * per + j < S serially (a thread past the end owns none and its
    total is 0), then the block scan of inner_cdf.  When 256 divides S this is inner_cdf's layout exactly; otherwise it
    equals inner_cdf of the weights padded with zeros to 256 * per entries (adding an exact 0 changes no sum)."""
    R, n = w.shape
    per = -(-n // LOSS_THREADS)
    pos = torch.arange(LOSS_THREADS, device=w.device)[:, None] * per + torch.arange(per, device=w.device)   # [256, per]
    own = pos < n
    wv = torch.where(own, w.float()[:, pos.clamp_max(n - 1)], torch.zeros((), device=w.device))             # [R, 256, per]
    run = torch.zeros(R, LOSS_THREADS, dtype=torch.float32, device=w.device)
    loc = torch.empty_like(wv)
    for j in range(per):
        run = torch.where(own[:, j], run + wv[:, :, j], run)
        loc[:, :, j] = run
    return (loc + _scan_base(run)[:, :, None]).reshape(R, LOSS_THREADS * per)[:, :n]


def _ulp(x: torch.Tensor) -> torch.Tensor:
    return torch.nextafter(x.abs(), torch.full_like(x, float("inf"))) - x.abs()


def inner_draw(cdf: torch.Tensor, seed: int, b_of: torch.Tensor, s_in_of: torch.Tensor, IR: int, ulps: int = 2):
    """The kernel's 3-of-n_s draw for hypotheses 0 .. IR-1 of every set (row of cdf).  b_of / s_in_of: int64 [S] pair
    and stream-in-pair of each row.  Returns (idx int64 [S, IR, 3], ambiguous bool [S, IR]); a hypothesis is ambiguous
    when a decision (the cdf search or a skip) compared values within `ulps` ulp of each other."""
    S, n = cdf.shape
    dev = cdf.device
    flat = cdf.reshape(-1)
    h = torch.arange(IR, dtype=torch.int64, device=dev)
    r = philox(h[None, :], s_in_of[:, None].to(dev), b_of[:, None].to(dev), INNER_TAG, seed ^ INNER_SEED_XOR)
    u = [(((r[k] >> 8).float() + 0.5) * 2.0 ** -24).reshape(-1) for k in range(3)]     # exact in fp32
    row = (torch.arange(S, device=dev) * n).repeat_interleave(IR)                       # [S * IR] offset of each row

    def at(i):                                                                          # cdf[i]
        return flat[row + i]

    def entry(i):                                                                       # (cdf[i], cdf[i] - cdf[i-1])
        hi = at(i)
        return hi, hi - torch.where(i > 0, at((i - 1).clamp_min(0)), torch.zeros_like(hi))

    def near(a, b_):
        return (a - b_).abs() <= ulps * torch.maximum(_ulp(a), _ulp(b_))

    W = at(torch.full_like(row, n - 1))
    clampW = W * torch.tensor(F32_ONE_MINUS_ULP, dtype=torch.float32, device=dev)
    removed = torch.zeros_like(W)
    amb = torch.zeros(S * IR, dtype=torch.bool, device=dev)
    ids = []
    for k in range(3):
        target = u[k] * (W - removed)
        if k > 0:
            skips = [ids[0]] if k == 1 else [torch.minimum(ids[0], ids[1]), torch.maximum(ids[0], ids[1])]
            for x in skips:                                             # skip drawn mass, in ascending index order
                hi, ex = entry(x)
                edge = hi - ex
                amb |= near(target, edge)
                target = torch.where(target >= edge, target + ex, target)
        tq = torch.minimum(target, clampW)
        lo = torch.zeros_like(row)
        hi_i = torch.full_like(row, n - 1)
        for _ in range(math.ceil(math.log2(n)) + 1):                   # first i with cdf[i] > tq (the kernel's search)
            act = lo < hi_i
            mid = (lo + hi_i) >> 1
            right = at(mid) > tq
            hi_i = torch.where(act & right, mid, hi_i)
            lo = torch.where(act & ~right, mid + 1, lo)
        pick = lo
        amb |= near(tq, at(pick)) | ((pick > 0) & near(tq, at((pick - 1).clamp_min(0))))
        for _ in range(3):                                              # the guard
            same = torch.zeros_like(amb)
            if k > 0:
                same |= pick == ids[0]
            if k > 1:
                same |= pick == ids[1]
            pick = torch.where(same, (pick + 1) % n, pick)
        ids.append(pick)
        removed = removed + entry(pick)[1]
    return torch.stack(ids, 1).reshape(S, IR, 3), amb.reshape(S, IR)


def loss_inner_draw(cdf: torch.Tensor, seed: int, b_of: torch.Tensor, s_in_of: torch.Tensor, IR: int, C: int,
                    ulps: int = 2, tag: int = LOSS_INNER_TAG, skip_in_draw_order: bool = False):
    """The training loss's C-of-n draw (loss_hyp_kernel) for hypotheses 0 .. IR-1 of every set (row of cdf, from
    loss_inner_cdf).  Draw k uses word k % 4 of Philox(seed ^ 0x9E3779B97F4A7C15)(h, s_in, b, tag + k / 4); its target
    u (W - removed) skips the mass of the entries drawn so far in ascending index order, is clamped to W (1 - 2^-24), and
    the first cdf entry above it is taken; the guard then advances a pick that was already drawn, cyclically, up to C
    times.  Returns (idx int64 [R, IR, C] in draw order, ambiguous bool [R, IR], as in inner_draw).  `tag` and
    `skip_in_draw_order` exist to plant mutations."""
    R, n = cdf.shape
    dev = cdf.device
    flat = cdf.reshape(-1)
    h = torch.arange(IR, dtype=torch.int64, device=dev)
    words = []
    for q in range(-(-C // 4)):
        r = philox(h[None, :], s_in_of[:, None].to(dev), b_of[:, None].to(dev), tag + q, seed ^ INNER_SEED_XOR)
        words += [x.reshape(-1) for x in r]
    row = (torch.arange(R, device=dev) * n).repeat_interleave(IR)

    def at(i):
        return flat[row + i]

    def entry(i):
        hi = at(i)
        return hi, hi - torch.where(i > 0, at((i - 1).clamp_min(0)), torch.zeros_like(hi))

    def near(a, b_):
        return (a - b_).abs() <= ulps * torch.maximum(_ulp(a), _ulp(b_))

    W = at(torch.full_like(row, n - 1))
    clampW = W * torch.tensor(F32_ONE_MINUS_ULP, dtype=torch.float32, device=dev)
    removed = torch.zeros_like(W)
    amb = torch.zeros(R * IR, dtype=torch.bool, device=dev)
    ids = []
    for k in range(C):
        u = ((words[k] >> 8).float() + 0.5) * 2.0 ** -24                               # u01_from_bits, in fp32
        target = u * (W - removed)
        if k > 0:
            prev = torch.stack(ids, 1)
            for x in (prev if skip_in_draw_order else prev.sort(1).values).unbind(1):
                hi, ex = entry(x)
                edge = hi - ex
                amb |= near(target, edge)
                target = torch.where(target >= edge, target + ex, target)
        tq = torch.minimum(target, clampW)
        lo = torch.zeros_like(row)
        hi_i = torch.full_like(row, n - 1)
        for _ in range(math.ceil(math.log2(n)) + 1):
            act = lo < hi_i
            mid = (lo + hi_i) >> 1
            right = at(mid) > tq
            hi_i = torch.where(act & right, mid, hi_i)
            lo = torch.where(act & ~right, mid + 1, lo)
        pick = lo
        amb |= near(tq, at(pick)) | ((pick > 0) & near(tq, at((pick - 1).clamp_min(0))))
        if k > 0:
            for _ in range(C):                                                          # the guard
                pick = torch.where((prev == pick[:, None]).any(1), (pick + 1) % n, pick)
        ids.append(pick)
        removed = removed + entry(pick)[1]
    return torch.stack(ids, 1).reshape(R, IR, C), amb.reshape(R, IR)


def inner_draw_check(got: torch.Tensor, want: torch.Tensor, amb: torch.Tensor) -> dict:
    """Kernel inner draws [R, IR, C] against loss_inner_draw's: `ok` when every hypothesis that differs is ambiguous."""
    diff = (got.to(want.device, torch.int64) != want).any(-1)
    bad = diff & ~amb
    return {"ok": int(bad.sum()) == 0, "n_bad": int(bad.sum()), "n_diff": int(diff.sum()), "n_amb": int(amb.sum())}


# ---------------------------------------------------------------------------------------------------------------
# the law of successive sampling
# ---------------------------------------------------------------------------------------------------------------
def law3(w) -> dict:
    """P({a, b, c}) = sum over the 6 orders of w_a / W * w_b / (W - w_a) * w_c / (W - w_a - w_b), for the positive
    entries of w (fp64).  Keys are ascending index triples."""
    w = [float(x) for x in w]
    pos = [i for i, x in enumerate(w) if x > 0]
    W = math.fsum(w[i] for i in pos)
    out = {}
    for tri in itertools.combinations(pos, 3):
        pr = 0.0
        for a, b, c in itertools.permutations(tri):
            pr += w[a] / W * w[b] / (W - w[a]) * w[c] / (W - w[a] - w[b])
        out[tri] = pr
    return out


def law3_with_replacement(w) -> dict:
    """Three independent draws ~ w, conditioned on three distinct entries: the law a draw with replacement would have."""
    w = [float(x) for x in w]
    pos = [i for i, x in enumerate(w) if x > 0]
    W = math.fsum(w[i] for i in pos)
    raw = {tri: 6.0 * w[tri[0]] * w[tri[1]] * w[tri[2]] / W ** 3 for tri in itertools.combinations(pos, 3)}
    z = math.fsum(raw.values())
    return {k: v / z for k, v in raw.items()}


def chi2_pvalue(counts: dict, law: dict, min_expected: float = 5.0) -> float:
    """Pearson chi^2 of observed triple counts against a law; bins expected below `min_expected` are pooled, and any
    triple outside the law's support makes the p-value 0."""
    from scipy.stats import chi2
    if any(k not in law for k in counts):
        return 0.0
    n = sum(counts.values())
    stat, dof, pool_o, pool_e = 0.0, -1, 0.0, 0.0
    for k, pk in law.items():
        e, o = n * pk, counts.get(k, 0)
        if e < min_expected:
            pool_o += o; pool_e += e
            continue
        stat += (o - e) ** 2 / e; dof += 1
    if pool_e > 0:
        stat += (pool_o - pool_e) ** 2 / pool_e; dof += 1
    return float(chi2.sf(stat, max(dof, 1)))


# ---------------------------------------------------------------------------------------------------------------
# the failure contract: which edge matrices torch.multinomial (and so the reference) refuses
# ---------------------------------------------------------------------------------------------------------------
CONTRACT_N, CONTRACT_B, CONTRACT_PAIR = 64, 4, 2          # 4096 cells per pair; the edge sits in pair 2 of 4
# case -> "zero" (torch.multinomial raises: the whole batch gets R = 0, t = 0, inliers = 0) or "pose"
CONTRACT = {
    "pos0": "zero", "pos1": "pose", "pos2": "pose", "pos3": "pose", "pos2047": "pose",
    "nan": "zero", "neg_nan": "zero", "inf": "zero", "negative": "zero", "neg_zero": "pose", "subnormal": "pose",
}


def contract_matrix(case: str, seed: int = 0) -> torch.Tensor:
    """final_scores [4, 64, 64] fp32: pairs 0, 1, 3 regular (every cell positive), pair 2 the edge case."""
    g = torch.Generator().manual_seed(seed)
    N, B = CONTRACT_N, CONTRACT_B
    fs = torch.rand(B, N, N, generator=g) * 1e-3 + 1e-6
    e = fs[CONTRACT_PAIR].view(-1)
    perm = torch.randperm(N * N, generator=g)
    if case.startswith("pos"):
        k = int(case[3:])
        e.zero_()
        e[perm[:k]] = torch.rand(k, generator=g) * 1e-3 + 1e-6
    elif case == "neg_nan":
        e.view(torch.int32)[perm[0]] = 0xFFC00001 - (1 << 32)         # a NaN with the sign bit set
    elif case in ("nan", "inf", "negative", "neg_zero"):
        e[perm[0]] = {"nan": float("nan"), "inf": float("inf"), "negative": -1e-6, "neg_zero": -0.0}[case]
    elif case == "subnormal":
        e.copy_(torch.rand(N * N, generator=g) * 1e-39 + 1e-41)      # every cell positive and below 2^-129 = 1.47e-39
    else:
        raise KeyError(case)
    return fs


def contract_geometry(seed: int = 1):
    """kps [4, 2, 64] in a 112x112 image, depths in [1, 2], K: the rest of a solver batch for `contract_matrix`."""
    g = torch.Generator().manual_seed(seed)
    N, B = CONTRACT_N, CONTRACT_B
    kps0 = torch.rand(B, 2, N, generator=g) * 112
    kps1 = torch.rand(B, 2, N, generator=g) * 112
    d0 = torch.rand(B, 1, N, generator=g) + 1
    d1 = torch.rand(B, 1, N, generator=g) + 1
    K = torch.tensor([[[100.0, 0, 56], [0, 100.0, 56], [0, 0, 1]]]).repeat(B, 1, 1)
    return kps0, d0, kps1, d1, K
