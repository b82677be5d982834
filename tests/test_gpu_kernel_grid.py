"""The GEMM family and the attention kernel, element by element against fp64, over the case table of
tests/kernel_grid.py: every launch regime and ring depth, every K residue of each ring, persistent grids with full and
partial last rounds, M tails, both group orders, every epilogue, and the attention kernel's query- and key-tile edges.

Each output buffer is filled with a sentinel first: rows past M, columns between N and the leading dimension and the
gaps between groups must keep it bit for bit.  Each check plants mutations of its reference -- the last tile (which runs
in the last persistent round) with its last K chunk dropped, that tile given the accumulators of the tile the same CTA
ran one round earlier, a 32-column chunk of the next row, for CONV the centre tap read one padded row off, for
attention the last key tile dropped, a key of the neighbouring image admitted and a query row of the next 192-row tile
-- and asserts that the bound rejects every one.  A failure names the case, the GEMM tile and its persistent round.
The bounds are those of tests/elementwise.py.  max(err / bound) per family and regime goes to $MICKEY_STAGE_METRICS."""
import math
import zlib

import pytest
import torch

from mickey_b200 import _lib
from tests import elementwise as ew
from tests import kernel_grid as kg
from tests.gpu_util import gemm, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = -7.25                      # exact in fp16 and fp32
_WORST: dict = {}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cases(epis):
    cases = [c for c in kg.gemm_cases(_sms()) if c.epi in epis]
    for c in cases:
        assert c.launch.regime == c.want, (c.name, c.launch.describe())
    return cases


def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def _randn(shape, seed, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def _record(family, regime, ratio):
    key = (family, regime)
    _WORST[key] = max(_WORST.get(key, 0.0), ratio)
    ew.record(family, f"kernel grid, {regime}", _WORST[key])


def _assert_sentinels(name, buf, written):
    """Every element of buf outside `written` still holds SENT, bit for bit."""
    itype = torch.int16 if buf.dtype == torch.float16 else torch.int32
    sent = torch.tensor([SENT], dtype=buf.dtype, device=DEV).view(itype)
    changed = (buf.view(itype) != sent) & ~written
    if bool(changed.any()):
        idx = changed.nonzero()[0].tolist()
        raise AssertionError(f"{name}: {int(changed.sum())} sentinel elements overwritten, first at {idx} "
                             f"(buffer {tuple(buf.shape)})")


def _run_all(cases, fn):
    """Run every case; report all failures together (each names its case, tile and round)."""
    failures = []
    for c in cases:
        try:
            fn(c)
        except AssertionError as e:
            failures.append(f"[{c.name}, {c.launch.describe()}] {e}")
    assert not failures, "\n".join(failures)


def _where(L, g):
    return ew.Where(lambda idx, g=g: (int(idx[0]), g, int(idx[1])), ew.Rows(), L)


def _pick_row(ok, start):
    """A row r >= start (or the last such before it) with ok[r] and ok[r + 1]."""
    n = ok.shape[0]
    both = (ok[:-1] & ok[1:]).nonzero().flatten()
    after = both[both >= min(start, n - 2)]
    return int(after[0]) if len(after) else int(both[-1])


def _tile_mutations(L, g, pres, post, drop, ref, ok=None):
    """Mutations of group g's reference ([M, N], rows are output rows): the last tile with its last K chunk dropped,
    the last tile given the previous round's tile of the same CTA, a 32-column chunk of the next row."""
    t, tp = L.mutation_tiles()
    gt, m0, n0 = L.tile(t)
    if gt != g:
        return []
    rows, cols = min(128, L.M - m0), min(L.bn, L.N - n0)
    rs, cs = slice(m0, m0 + rows), slice(n0, n0 + cols)
    muts = [ew.Mutation(f"K chunk {L.k_chunks - 1} dropped from tile {t} (round {t // L.grid})", (rs, cs),
                        post(pres[g][rs, cs] - drop(g, rs, cs), rs, cs))]
    if tp is not None:
        gp, mp, np_ = L.tile(tp)
        r2, c2 = min(rows, L.M - mp), min(cols, L.N - np_)
        rs2, cs2 = slice(m0, m0 + r2), slice(n0, n0 + c2)
        muts.append(ew.Mutation(f"tile {t} given the accumulators of tile {tp} (round {tp // L.grid})", (rs2, cs2),
                                post(pres[gp][mp:mp + r2, np_:np_ + c2], rs2, cs2)))
    if L.M >= 2:
        ok = torch.ones(L.M, dtype=torch.bool, device=DEV) if ok is None else ok
        r = _pick_row(ok, m0 + 5)
        muts.append(ew.row_chunk_swap(ref, r, n0, min(32, L.N - n0)))
    return muts


def _check(family, c, impl, name, got, ref, bound, where, muts, regime):
    r = ew.check(f"{c.name} {impl} {name}", got, ref, bound.clamp_min(1e-30), where, muts)
    _record(family, regime, r)
    return len(muts)


# ---------------------------------------------------------------------------------------------------------------
# STORE_H / STORE_F / RESID_F, grouped or not
# ---------------------------------------------------------------------------------------------------------------
def _a_g(c, A, g):
    r0, c0 = g * c.a_row_group_off, c.a_col_base + g * c.a_col_group_off
    return A[r0:r0 + c.M, c0:c0 + c.K]


def _b_g(c, B, g):
    return B[g * c.b_row_group_off:g * c.b_row_group_off + c.N]


def _operands(c, seed):
    A = _randn(((c.groups - 1) * c.a_row_group_off + c.M, c.a_col_base + (c.groups - 1) * c.a_col_group_off + c.K), seed)
    B = _randn(((c.groups - 1) * c.b_row_group_off + c.N, c.K), seed + 1, 1 / math.sqrt(c.K))
    return A, B


def _products(c, A, B):
    pres, abss = [], []
    for g in range(c.groups):
        a, b = _a_g(c, A, g).double(), _b_g(c, B, g).double()
        pres.append(a @ b.t())
        abss.append(a.abs() @ b.abs().t())
    return pres, abss


def _linear_case(c):
    L, M, N, G, K = c.launch, c.M, c.N, c.groups, c.K
    seed = _seed(c.name)
    A, B = _operands(c, seed)
    bias = _randn((G * N,), seed + 2, 0.1, torch.float32) if c.bias else None
    gamma = _randn((N,), seed + 3, 1.0, torch.float32)
    x0 = _randn((M, N), seed + 4, 1.0, torch.float32)
    pres, abss = _products(c, A, B)
    gs = N + 32
    ld = G * gs + 32
    rows = L.m_tiles * 128 + 8
    fp16 = c.epi == "STORE_H"
    refs, bounds, posts = [], [], []
    for g in range(G):
        pre = pres[g]
        b = bias[g * N:(g + 1) * N].double() if bias is not None else torch.zeros(N, dtype=torch.float64, device=DEV)
        acc = ew.gemm_acc_bound(K, abss[g])
        gm, x0d = gamma.double(), x0.double()

        def post(p, rs, cs, b=b, gm=gm, x0d=x0d):
            if c.epi == "STORE_F":
                return p
            if c.epi == "RESID_F":
                return x0d[rs, cs] + gm[cs] * (p + b[cs])
            t = p + b[cs]
            return ew.gelu64(t) if c.act == 1 else t.relu() if c.act == 2 else t

        allr = slice(None)
        ref = post(pre, allr, allr)
        if c.epi == "STORE_F":
            bound = acc + ew.out_rounding(ref, False)
        elif c.epi == "RESID_F":
            bound = gm.abs() * (acc + ew.epilogue_terms(pre, b)) + ew.epilogue_terms(ref, x0d) + ew.out_rounding(ref, False)
        else:
            e = acc + ew.epilogue_terms(pre, b)
            bound = (ew.gelu_bound(pre + b, e) if c.act == 1 else e) + ew.out_rounding(ref, True)
        refs.append(ref), bounds.append(bound), posts.append(post)

    def drop(g, rs, cs):
        return _a_g(c, A, g)[rs, K - 64:K].double() @ _b_g(c, B, g)[cs, K - 64:K].double().t()

    impls = ("tc", "simt")
    for impl in impls:
        buf = torch.full((rows, ld), SENT, dtype=torch.float16 if fp16 else torch.float32, device=DEV)
        kw = dict(groups=G, a_row_group_off=c.a_row_group_off, a_col_group_off=c.a_col_group_off, a_col_base=c.a_col_base,
                  b_row_group_off=c.b_row_group_off)
        if c.epi == "STORE_H":
            kw.update(out_h=buf, out_h_ld=ld, out_h_group_off=gs, act=c.act)
            if bias is not None:
                kw.update(bias=bias, bias_group_off=N)
        elif c.epi == "STORE_F":
            kw.update(out_f=buf, out_f_ld=ld, out_f_group_off=gs)
        else:
            assert G == 1
            buf[:M, :N] = x0
            kw.update(out_f=buf, out_f_ld=ld, bias=bias, gamma=gamma)
        gemm(c.epi, A, B, M, N, K, impl=impl, **kw)
        torch.cuda.synchronize()
        written = torch.zeros_like(buf, dtype=torch.bool)
        for g in range(G):
            written[:M, g * gs:g * gs + N] = True
        _assert_sentinels(f"{impl} output", buf, written)
        planted = 0
        for g in range(G):
            muts = _tile_mutations(L, g, pres, posts[g], drop, refs[g])
            planted += _check(c.epi, c, impl, f"group {g}", buf[:M, g * gs:g * gs + N], refs[g], bounds[g], _where(L, g),
                              muts, L.regime)
        assert planted >= 2, "no mutation planted"


def test_gemm_regime_grid():
    """STORE_H (act none / GELU / ReLU, with and without bias), STORE_F and RESID_F (in place, LayerScale) over every
    regime x BN x K residue cell, the persistent round shapes, the cutovers and the M tails; both group orders."""
    _run_all(_cases(("STORE_H", "STORE_F", "RESID_F")), _linear_case)


# ---------------------------------------------------------------------------------------------------------------
# PATCH
# ---------------------------------------------------------------------------------------------------------------
def _patch_case(c):
    L, M, N, K = c.launch, c.M, c.N, c.K
    tok = c.extra["tok_per_img"]
    n_img = M // tok
    seed = _seed(c.name)
    P = _randn((M, K), seed)
    W = _randn((N, K), seed + 1, 1 / math.sqrt(K))
    posb = _randn((tok, N), seed + 2, 1.0, torch.float32)
    m = torch.arange(M, device=DEV)
    orow = (m // tok) * (tok + 1) + 1 + m % tok
    pre = P.double() @ W.double().t()
    pe = posb.double()[m % tok]
    ref = pre + pe
    bound = ew.gemm_acc_bound(K, P.double().abs() @ W.double().abs().t()) + ew.epilogue_terms(pre, pe) + ew.out_rounding(ref, False)

    def post(p, rs, cs):
        return p + pe[rs, cs]

    def drop(g, rs, cs):
        return P[rs, K - 64:].double() @ W[cs, K - 64:].double().t()

    where = ew.Where(lambda idx: (int(idx[0]), 0, int(idx[1])), ew.Rows("patches", tok), L)
    for impl in ("tc", "simt"):
        buf = torch.full((n_img * (tok + 1) + 8, N + 32), SENT, device=DEV)
        gemm("PATCH", P, W, M, N, K, impl=impl, aux=posb, tok_per_img=tok, out_f=buf, out_f_ld=N + 32)
        torch.cuda.synchronize()
        written = torch.zeros_like(buf, dtype=torch.bool)
        written[orow, :N] = True
        _assert_sentinels(f"{impl} token matrix (cls rows, pad columns, rows past the last image)", buf, written)
        muts = _tile_mutations(L, 0, [pre], post, drop, ref)
        muts.append(ew.Mutation("token of the neighbouring image", (slice(tok + 3, tok + 4),), ref[3:4]))
        _check("PATCH", c, impl, "X", buf[orow, :N], ref, bound, where, muts, L.regime)


def test_gemm_patch_embedding():
    _run_all(_cases(("PATCH",)), _patch_case)


# ---------------------------------------------------------------------------------------------------------------
# CONV
# ---------------------------------------------------------------------------------------------------------------
def _conv_case(c):
    L, ex = c.launch, c.extra
    n_img, h2, w2, cin, G, pad = ex["n_img"], ex["h2"], ex["w2"], ex["cin"], ex["G"], ex["pad"]
    R, cout, cpt = c.M, c.N, ex["cin"] // 64
    assert R == n_img * h2 * w2 and c.k_chunks == 9 * cpt and c.act in (0, 2)
    mask = ex.get("mask", 0)
    seed = _seed(c.name)
    A = _randn((R, G * cin), seed)
    Wt = _randn((G * cout, 9 * cin), seed + 1, 1 / math.sqrt(9 * cin))
    bias = _randn((G * cout,), seed + 2, 0.1, torch.float32) if c.bias else None
    res = _randn((R, G * cout), seed + 3) if pad else None
    pe = _randn((h2 * w2, cout), seed + 4, 1.0, torch.float32) if pad else None
    shifts = [(ky - 1) * w2 + (kx - 1) for ky in range(3) for kx in range(3)]
    halo = w2 + 1
    per = h2 * w2
    pos = torch.arange(R, device=DEV) % per
    y, x = pos // w2, pos % w2
    valid = ((y >= 1) & (y <= h2 - 2) & (x >= 1) & (x <= w2 - 2)) if pad else torch.ones(R, dtype=torch.bool, device=DEV)
    slabs, pres, refs, bounds, posts = [], [], [], [], []
    for g in range(G):
        slab = torch.zeros(R + 2 * halo, cin, dtype=torch.float64, device=DEV)       # TMA zero fill outside the tensor
        slab[halo:halo + R] = A[:, g * cin:(g + 1) * cin].double()
        Wd = Wt[g * cout:(g + 1) * cout].double()
        pre = torch.zeros(R, cout, dtype=torch.float64, device=DEV)
        ab = torch.zeros_like(pre)
        for t, s in enumerate(shifts):
            a = slab[halo + s:halo + s + R]
            w = Wd[:, t * cin:(t + 1) * cin]
            pre += a @ w.t()
            ab += a.abs() @ w.abs().t()
        b = bias[g * cout:(g + 1) * cout].double() if bias is not None else torch.zeros(cout, dtype=torch.float64, device=DEV)
        rg = res[:, g * cout:(g + 1) * cout].double() if res is not None else torch.zeros_like(pre)
        pe_t = pe.double()[pos] if (pe is not None and (mask >> g) & 1) else None

        def post(p, rs, cs, b=b, rg=rg, pe_t=pe_t):
            t = p + b[cs] + rg[rs, cs]
            t = t.relu() if c.act == 2 else t
            if pe_t is not None:
                t = t + pe_t[rs, cs]
            return torch.where(valid[rs, None], t, torch.zeros_like(t))

        allr = slice(None)
        ref = post(pre, allr, allr)
        bound = ew.gemm_acc_bound(9 * cin, ab) + ew.epilogue_terms(pre, b, rg, pe_t, ref)
        bound = torch.where(valid[:, None], bound, torch.zeros_like(bound))
        slabs.append(slab), pres.append(pre), refs.append(ref), bounds.append(bound), posts.append(post)

    kc = c.k_chunks - 1
    tap, kin = divmod(kc, cpt)

    def drop(g, rs, cs):
        a = slabs[g][halo + shifts[tap] + rs.start:halo + shifts[tap] + rs.stop, kin * 64:(kin + 1) * 64]
        return a @ Wt[g * cout + cs.start:g * cout + cs.stop, tap * cin + kin * 64:tap * cin + (kin + 1) * 64].double().t()

    gsf, gsh = cout + 32, 2 * cout
    taps_kw = dict(taps=shifts, chunks_per_tap=cpt, groups=G, a_col_group_off=c.a_col_group_off,
                   b_row_group_off=c.b_row_group_off, act=c.act)
    if bias is not None:
        taps_kw.update(bias=bias, bias_group_off=cout)
    if pad:
        taps_kw.update(res_h=res, res_h_ld=G * cout, res_h_group_off=cout, pad_h2=h2, pad_w2=w2, aux=pe, aux_group_mask=mask)
    for impl in ("tc", "simt"):
        oh = torch.full((L.m_tiles * 128 + 8, G * gsh), SENT, dtype=torch.float16, device=DEV)
        of = torch.full((L.m_tiles * 128 + 8, G * gsf + 32), SENT, device=DEV) if pad else None
        kw = dict(taps_kw, out_h=oh, out_h_ld=G * gsh, out_h_group_off=gsh)
        if of is not None:
            kw.update(out_f=of, out_f_ld=G * gsf + 32, out_f_group_off=gsf)
        gemm("CONV", A, Wt, R, cout, impl=impl, **kw)
        torch.cuda.synchronize()
        for buf, gsz, what in ((oh, gsh, "fp16"), (of, gsf, "fp32")):
            if buf is None:
                continue
            written = torch.zeros_like(buf, dtype=torch.bool)
            for g in range(G):
                written[:R, g * gsz:g * gsz + cout] = True
            _assert_sentinels(f"{impl} {what} output", buf, written)
            planted = 0
            for g in range(G):
                muts = _tile_mutations(L, g, pres, posts[g], drop, refs[g], valid)
                if muts:
                    _, m0, _ = L.tile(L.mutation_tiles()[0])
                    r = _pick_row(valid, m0 + 3)
                    w4 = Wt[g * cout:(g + 1) * cout, 4 * cin:5 * cin].double()
                    pm = pres[g][r:r + 1] - slabs[g][halo + r:halo + r + 1] @ w4.t() + slabs[g][halo + r + w2:halo + r + w2 + 1] @ w4.t()
                    muts.append(ew.Mutation("centre tap read one padded row off", (slice(r, r + 1), slice(None)),
                                            posts[g](pm, slice(r, r + 1), slice(None))))
                bd = bounds[g] + torch.where(valid[:, None], ew.out_rounding(refs[g], what == "fp16"), torch.zeros_like(refs[g]))
                planted += _check(f"CONV {what}", c, impl, f"{what} group {g}", buf[:R, g * gsz:g * gsz + cout], refs[g], bd,
                                  ew.Where(lambda idx, g=g: (int(idx[0]), g, int(idx[1])), ew.Rows("padded", per, w2), L),
                                  muts, L.regime)
            assert planted >= 3, "no mutation planted"


def test_gemm_conv_epilogue():
    """3x3 shifted-row convolutions: taps off both ends of the tensor (zero fill), the pad ring zeroed, the fp16
    shortcut, the PE on the groups of each aux_group_mask, fp32 and fp16 outputs from the same launch."""
    _run_all(_cases(("CONV",)), _conv_case)


# ---------------------------------------------------------------------------------------------------------------
# LN (grouped, N = 128, fp32 residual, pad mask)
# ---------------------------------------------------------------------------------------------------------------
def _ln_case(c):
    L, M, G, K, ex = c.launch, c.M, c.groups, c.K, c.extra
    h2, w2 = ex["h2"], ex["w2"]
    per = h2 * w2
    seed = _seed(c.name)
    A, B = _operands(c, seed)
    gam = _randn((G * 128,), seed + 2, 1.0, torch.float32)
    bet = _randn((G * 128,), seed + 3, 0.3, torch.float32)
    x0 = _randn((M, G * 128), seed + 4, 1.0, torch.float32)
    pos = torch.arange(M, device=DEV) % per
    y, x = pos // w2, pos % w2
    valid = (y >= 1) & (y <= h2 - 2) & (x >= 1) & (x <= w2 - 2)
    pres, abss = _products(c, A, B)
    refs, bounds, posts = [], [], []
    for g in range(G):
        gm, bt = gam[g * 128:(g + 1) * 128].double(), bet[g * 128:(g + 1) * 128].double()
        xg = x0[:, g * 128:(g + 1) * 128].double()
        yv, b = ew.ln_bound(pres[g], ew.gemm_acc_bound(K, abss[g]), gm, bt, 1e-5)
        ref = torch.where(valid[:, None], xg + yv, torch.zeros_like(yv))
        bound = torch.where(valid[:, None], b + ew.epilogue_terms(xg, yv, ref), torch.zeros_like(b))

        def post(p, rs, cs, gm=gm, bt=bt, xg=xg):
            assert cs == slice(0, 128) or cs == slice(None)
            t = xg[rs] + ew.ln_bound(p, 0.0, gm, bt, 1e-5)[0]
            return torch.where(valid[rs, None], t, torch.zeros_like(t))

        refs.append(ref), bounds.append(bound), posts.append(post)

    def drop(g, rs, cs):
        return _a_g(c, A, g)[rs, K - 64:K].double() @ _b_g(c, B, g)[cs, K - 64:K].double().t()

    gsf, gsh = 160, 256
    for impl in ("tc", "simt"):
        of = torch.full((L.m_tiles * 128 + 8, G * gsf + 32), SENT, device=DEV)
        oh = torch.full((L.m_tiles * 128 + 8, G * gsh), SENT, dtype=torch.float16, device=DEV)
        for g in range(G):
            of[:M, g * gsf:g * gsf + 128] = x0[:, g * 128:(g + 1) * 128]
        gemm("LN", A, B, M, 128, K, impl=impl, groups=G, a_row_group_off=c.a_row_group_off, a_col_group_off=c.a_col_group_off,
             a_col_base=c.a_col_base, b_row_group_off=c.b_row_group_off, gamma=gam, beta=bet, ln_group_off=128, eps=1e-5,
             out_f=of, out_f_ld=G * gsf + 32, out_f_group_off=gsf, out_h=oh, out_h_ld=G * gsh, out_h_group_off=gsh,
             pad_h2=h2, pad_w2=w2)
        torch.cuda.synchronize()
        for buf, gsz, fp16 in ((of, gsf, False), (oh, gsh, True)):
            written = torch.zeros_like(buf, dtype=torch.bool)
            for g in range(G):
                written[:M, g * gsz:g * gsz + 128] = True
            _assert_sentinels(f"{impl} {'fp16' if fp16 else 'fp32'} output", buf, written)
            planted = 0
            for g in range(G):
                muts = _tile_mutations(L, g, pres, posts[g], drop, refs[g], valid)
                bd = bounds[g] + torch.where(valid[:, None], ew.out_rounding(refs[g], fp16), torch.zeros_like(refs[g]))
                planted += _check("LN", c, impl, f"{'fp16' if fp16 else 'fp32'} group {g}", buf[:M, g * gsz:g * gsz + 128],
                                  refs[g], bd, ew.Where(lambda idx, g=g: (int(idx[0]), g, int(idx[1])),
                                                        ew.Rows("padded", per, w2), L), muts, L.regime)
            assert planted >= 2, "no mutation planted"


def test_gemm_layernorm_epilogue():
    _run_all(_cases(("LN",)), _ln_case)


# ---------------------------------------------------------------------------------------------------------------
# the matcher: EPI_LSE -> mk_op_matcher_reduce -> EPI_DUAL
# ---------------------------------------------------------------------------------------------------------------
def _matcher_case(c, lse_case):
    ex, n, L = c.extra, c.M, c.launch
    Ll = lse_case.launch
    B, bound_mode, pitch, lean = ex["B"], ex["lse_bound"], ex["pitch"], ex["lean"]
    T, dust = 0.1, 1.0
    lib = _lib.load()
    seed = _seed(c.name)
    d0 = torch.nn.functional.normalize(_randn((B, n, 128), seed, 1.0, torch.float32), dim=-1)
    d1 = torch.nn.functional.normalize(_randn((B, n, 128), seed + 1, 1.0, torch.float32), dim=-1)
    g = torch.Generator(device=DEV).manual_seed(seed + 2)
    s0, s1 = torch.rand(B, n, generator=g, device=DEV), torch.rand(B, n, generator=g, device=DEV)

    def split(d, role):
        hi = d.half()
        lo = (d - hi.float()).half()
        return torch.cat([hi, lo, hi] if role == 0 else [hi, hi, lo], dim=-1).reshape(B * n, 384).contiguous()

    a0, a1 = split(d0, 0), split(d1, 1)
    npad = kg.cdiv(n, 128) * 128
    pr = torch.full((B, npad // 64, npad, 2), float("nan"), device=DEV)
    pc = torch.full((B, npad // 32, npad, 2), float("nan"), device=DEV)
    lr = torch.full((B, npad), SENT, device=DEV)
    lc = torch.full((B, npad), SENT, device=DEV)
    dust_t = torch.tensor([dust], device=DEV)
    common = dict(groups=B, a_row_group_off=n, b_row_group_off=n, n_valid=n, inv_temp=1 / T, part_ld=npad)
    gemm("LSE", a0, a1, n, n, 384, part_row=pr, part_col=pc, lse_bound=bound_mode, **common)
    _lib.check(lib.mk_op_matcher_reduce(_lib.ptr(pr), _lib.ptr(pc), _lib.ptr(dust_t), B, n, npad, _lib.ptr(lr), _lib.ptr(lc),
                                        stream()))
    size = B * n * pitch
    flats = [torch.full((size + 64,), SENT, device=DEV) for _ in range(1 if lean else 3)]
    views = [f[:size].view(B, n, pitch) for f in flats]
    kw = dict(final_scores=views[-1]) if lean else dict(scores=views[0], kp_scores=views[1], final_scores=views[2])
    gemm("DUAL", a0, a1, n, n, 384, lse_r=lr, lse_c=lc, scr0=s0, scr1=s1, out_pitch=pitch, **kw, **common)
    torch.cuda.synchronize()
    # sentinels: lse entries past n, the pad columns of every output row (a tensor store may zero columns n .. n4, the
    # values the kernel computes beyond n_valid), and what follows the last row
    written = torch.zeros(B, npad, dtype=torch.bool, device=DEV)
    written[:, :n] = True
    _assert_sentinels("lse_r", lr, written)
    _assert_sentinels("lse_c", lc, written)
    n4 = (n + 3) // 4 * 4 if L.out_tma else n
    for f, v in zip(flats, views):
        w = torch.zeros(size + 64, dtype=torch.bool, device=DEV)
        wv = w[:size].view(B, n, pitch)
        wv[:, :, :n] = True
        wv[:, :, n:n4] = v[:, :, n:n4] == 0
        _assert_sentinels("output", f, w)
    k2 = (1 / T) / math.log(2)
    dl = dust / math.log(2)
    U32 = ew.U32
    done = 0
    t_last, tp = L.mutation_tiles()
    g_last, m0, n0 = L.tile(t_last)
    rs = slice(m0, min(n, m0 + 128))
    cs = slice(n0, min(n, n0 + 128))
    # the lse vectors: the last LSE tile with all of its 128 x 128 cells valid (a 1 x 1 corner tile moves a row's
    # log-sum-exp by less than its bound)
    tl = next(t for t in range(Ll.tiles - 1, -1, -1)
              if all(min(128, n - o) == min(128, n) for o in Ll.tile(t)[1:]))
    gl, ml, nl = Ll.tile(tl)
    rl, cl = slice(ml, min(n, ml + 128)), slice(nl, min(n, nl + 128))
    Ss = []
    for p in range(B):
        a, b = a0[p * n:(p + 1) * n].double(), a1[p * n:(p + 1) * n].double()
        Ss.append(a @ b.t())
    for p in range(B):
        a, b = a0[p * n:(p + 1) * n].double(), a1[p * n:(p + 1) * n].double()
        S = Ss[p]
        x = S * k2
        dx = k2 * 384 * 2.0 ** -23 * (a.abs() @ b.abs().t()) + 2 * U32 * x.abs()
        xd = torch.full((1, 1), dl, dtype=torch.float64, device=DEV)

        def lse_rows(xx):
            return torch.logsumexp(torch.cat([xx, xd.expand(xx.shape[0], 1)], 1) * math.log(2), 1) / math.log(2)

        def lse_cols(xx):
            return torch.logsumexp(torch.cat([xx, xd.expand(1, xx.shape[1])], 0) * math.log(2), 0) / math.log(2)

        lr_ref, lc_ref = lse_rows(x), lse_cols(x)
        dlr = dx.amax(1) + ((n + 1) * U32 + 2.0 ** -22) / math.log(2) + 2.0 ** -22 * lr_ref.abs()
        dlc = dx.amax(0) + ((n + 1) * U32 + 2.0 ** -22) / math.log(2) + 2.0 ** -22 * lc_ref.abs()
        mr, mc = [], []
        chunk = None
        if p == g_last:
            chunk = a[rs, :64] @ b[cs, :64].t()            # hi.hi: chunks 2 and 5 only carry the lo corrections
        if p == gl:
            xm = x.clone()
            xm[rl, cl] -= k2 * (a[rl, :64] @ b[cl, :64].t())
            mr.append(ew.Mutation(f"K chunk 0 dropped from tile {tl} (round {tl // Ll.grid})", (rl,), lse_rows(xm[rl])))
            mc.append(ew.Mutation(f"K chunk 0 dropped from tile {tl} (round {tl // Ll.grid})", (cl,), lse_cols(xm[:, cl])))
        if n >= 2:
            mr.append(ew.Mutation("lse of the next row", (slice(0, 1),), lr_ref[1:2]))
            mc.append(ew.Mutation("lse of the next column", (slice(0, 1),), lc_ref[1:2]))
        r = ew.check(f"{c.name} lse_r pair {p}", lr[p, :n], lr_ref, dlr, mutations=mr)
        _record("matcher lse", Ll.regime, r)
        r = ew.check(f"{c.name} lse_c pair {p}", lc[p, :n], lc_ref, dlc, mutations=mc)
        _record("matcher lse", Ll.regime, r)
        rel = math.log(2) * (2 * dx + dlr[:, None] + dlc[None, :]) + 2.0 ** -22 + 4 * U32
        kp = s0[p].double()[:, None] * s1[p].double()[None, :]

        def score(Sb, r_, c_):
            return torch.exp2(2 * k2 * Sb - lr_ref[r_, None] - lc_ref[None, c_])

        sc_ref = score(S, slice(None), slice(None))
        f_ref = sc_ref * kp
        outs = [("final_scores", views[-1], f_ref, f_ref * (rel + 3 * U32) + 2.0 ** -126, lambda Sb, r_, c_: score(Sb, r_, c_) * kp[r_, c_])]
        if not lean:
            outs.append(("scores", views[0], sc_ref, sc_ref * rel + 2.0 ** -126, score))
            outs.append(("kp_scores", views[1], kp, U32 * kp + 2.0 ** -126, None))
        for what, v, ref, bd, post in outs:
            muts = []
            if post is not None and p == g_last:
                muts.append(ew.Mutation(f"K chunk 0 dropped from tile {t_last}", (rs, cs), post(S[rs, cs] - chunk, rs, cs)))
                if tp is not None:
                    gp, mp, np_ = L.tile(tp)
                    r2, c2 = min(rs.stop - rs.start, n - mp), min(cs.stop - cs.start, n - np_)
                    muts.append(ew.Mutation(f"tile {t_last} given the accumulators of tile {tp}",
                                            (slice(m0, m0 + r2), slice(n0, n0 + c2)),
                                            post(Ss[gp][mp:mp + r2, np_:np_ + c2], slice(m0, m0 + r2), slice(n0, n0 + c2))))
            if n >= 2:
                muts.append(ew.row_chunk_swap(ref, min(5, n - 2), 0, min(32, n)))
            r = ew.check(f"{c.name} {what} pair {p}", v[p, :, :n], ref, bd, ew.Where(lambda idx, p=p: (int(idx[0]), p, int(idx[1])), ew.Rows(), L), muts)
            _record(f"matcher {what}", L.regime, r)
            done += len(muts)
    assert done >= 2


def test_matcher_lse_reduce_dual():
    """n_valid = 2, 127, 128, 129 and 1938; fixed-shift and true-maxima partials; TMA tensor stores and st.global; lean
    mode.  EPI_LSE reaches the persistent grid at n_valid = 1938."""
    cases = _cases(("LSE", "DUAL"))
    lse = {c.name[4:]: c for c in cases if c.epi == "LSE"}
    _run_all([c for c in cases if c.epi == "DUAL"], lambda c: _matcher_case(c, lse[c.name[5:]]))


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
class _AttnWhere(ew.Where):
    def __init__(self, c):
        super().__init__()
        self.c = c

    def describe(self, idx):
        i, h, t, d = (int(v) for v in idx)
        c = self.c
        tile = (i * c.heads + h) * c.q_tiles + t // kg.ATTN_BQ
        return (f"image {i}, head {h}, query {t}, dim {d}; attention tile {tile} (query tile {t // kg.ATTN_BQ}), "
                f"round {tile // min(c.tiles, c.sms)} of {min(c.tiles, c.sms)} persistent CTAs")


def _attn_case(c, impl):
    lib = _lib.load()
    T, n_img, heads = c.T, c.n_img, c.heads
    D = heads * 64
    qkv = _randn((n_img * T, 3 * D), _seed(c.name), c.scale)
    n_kv = kg.cdiv(T, kg.ATTN_BK)
    h = heads - 1
    qv = qkv.view(n_img, T, 3, heads, 64)
    if n_kv >= 2:
        qv[0, 0, 0, h] = qv[0, T - 1, 1, h]      # query 0 of image 0 aimed at the last key: the last key tile carries weight
    if c.leak:
        qv[1::2, :, 1] = (qv[1::2, :, 1].float() * 50).half()
    out = torch.full((n_img * T + 256, D), SENT, dtype=torch.float16, device=DEV)
    _lib.check(lib.mk_op_attention(_lib.ptr(qkv), _lib.ptr(out), n_img, T, D, heads, impl, stream()))
    torch.cuda.synchronize()
    written = torch.zeros_like(out, dtype=torch.bool)
    written[:n_img * T] = True
    _assert_sentinels("rows past the last image", out, written)
    q, k, v = qkv.double().reshape(n_img, T, 3, heads, 64).permute(2, 0, 3, 1, 4)
    ref, bound = ew.attention_ref_bound(q, k, v)
    got = out[:n_img * T].reshape(n_img, T, heads, 64).permute(0, 2, 1, 3)
    muts = []
    if n_kv >= 2:
        cut = (n_kv - 1) * kg.ATTN_BK
        s = (q[0, h, :1] @ k[0, h].t()) * 0.125
        o = torch.softmax(s[:, :cut], -1) @ v[0, h, :cut]
        muts.append(ew.Mutation("last key tile dropped", (0, h, slice(0, 1)), o))
    cap = min(n_kv * kg.ATTN_BK, n_img * T)
    if c.leak and cap > T:
        # a key that the last key tile of image 0 reads past T (the next image's, scaled x50) admitted into the softmax
        # of the query row where it would weigh most
        kf = k[:, h].reshape(n_img * T, 64)[T:cap]
        vf = v[:, h].reshape(n_img * T, 64)[T:cap]
        own = (q[0, h] @ k[0, h].t()) * 0.125
        extra, j = ((q[0, h] @ kf.t()) * 0.125).max(1)
        pe = torch.softmax(torch.cat([own, extra[:, None]], 1), -1)
        r = int(pe[:, -1].argmax())
        o = pe[r] @ torch.cat([v[0, h], vf[int(j[r])][None]], 0)
        muts.append(ew.Mutation("a key of the neighbouring image admitted", (0, h, slice(r, r + 1)), o[None]))
    i = n_img - 1
    if T > kg.ATTN_BQ:
        r = min(5, T - kg.ATTN_BQ - 1)
        muts.append(ew.Mutation("query row of the next 192-row tile", (i, h, slice(r, r + 1)),
                                ref[i, h, r + kg.ATTN_BQ:r + kg.ATTN_BQ + 1]))
    name = {1: "wgmma", 2: "mma.sync"}[impl]
    r = ew.check(f"attention {name} {c.name}", got, ref, bound, _AttnWhere(c), muts)
    _record(f"attention {name}", c.grid, r)
    assert muts or T <= kg.ATTN_BK


@pytest.mark.parametrize("impl", [1, 2], ids=["wgmma", "mma_sync"])
def test_attention_grid(impl):
    """T across the 128-key and 192-query tile edges; grids of fewer tiles than SMs, exactly one per SM and a partial
    last round; logit scales at which the running maximum moves and P falls below fp16's normal range; every odd
    image's K scaled x50, so that a key read past T from the next image would dominate its row."""
    cases = kg.attention_cases(_sms())
    failures = []
    for c in cases:
        try:
            _attn_case(c, impl)
        except AssertionError as e:
            failures.append(f"[{c.name}: {c.n_img} images x {c.heads} heads, {c.tiles} tiles, {c.grid}] {e}")
    assert not failures, "\n".join(failures)
