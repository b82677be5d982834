"""The solver's two random draws against their definitions (restatements in tests/draws.py).

- Outer draw: every stream of a production batch (C3: ViT-B, 32 pairs, 16 x 64, final_scores at padded pitch 1952;
  C2: ViT-S, 1 pair; L: ViT-L, IM = 20, so the third Philox group is partly unused) is the fp64 exponential race's top
  2048 up to cells in the 1e-4 key band; the same through mk_op_sample in every addressing mode and at edge counts.
- Inner draw: every hypothesis's triple is restated bit for bit in fp32; its hyp_Rt and hyp_scores must match an fp64
  Kabsch and soft count of that triple, and the pose the fp64 oracle's with both draws injected.
- The failure contract: the zero pose exactly where torch.multinomial raises (the table in tests/draws.py).
- The inner law: 524 k hypotheses on a set whose hypotheses decode to their triples, chi^2 against the closed form.
Each check is shown to reject planted mutations.  Counts and p-values are printed (pytest -s) and quoted in DESIGN §2.
"""
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from oracle import mickey_oracle as mo
from tests import draws, stages
from tests.common import synthetic_pair
from tests.gpu_util import stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, W = 720, 540
N_S = 2048
GEOS = {"C3": ("vitb", 32, 16, 64), "C2": ("vits", 1, 8, 64), "L": ("vitl", 1, 20, 100)}
SEED = stages.SEED


def _model(variant, im, ir, seed=3):
    cfg = mickey_cfg(variant, im, ir)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=seed), strict=True)
    return cfg, model.cuda().eval()


class Prod(stages.Solved):
    """compute_matches at 720x540, then the solver with its own draws."""

    def __init__(self, name):
        variant, B, im, ir = GEOS[name]
        cfg, model = _model(variant, im, ir)
        data = {k: v.to(DEV) for k, v in synthetic_pair(B, H, W, seed=17).items()}
        with torch.no_grad():
            model.compute_matches(data)
        super().__init__(name, cfg, model, data, B, im, ir)


@pytest.fixture(scope="module", params=list(GEOS))
def prod(request):
    p = Prod(request.param)
    yield p
    del p
    torch.cuda.empty_cache()


def test_production_outer_draw_is_the_race(prod):
    if prod.name == "C3":
        assert prod.fs.stride(1) == 1952                    # the matcher's padded pitch: ROW_VEC loads
    stages.outer_draws_are_the_race(prod)


def test_production_inner_draws_are_restated(prod):
    stages.inner_draws_are_restated(prod)


# ---------------------------------------------------------------------------------------------------------------
# mk_op_sample: layouts, sizes and edge distributions
# ---------------------------------------------------------------------------------------------------------------
def _sample(fs, pitch, IM, seed):
    """fs [B, N, >= N] (row pitch `pitch` floats) -> (idx [B, IM, n_s], status)."""
    lib = _lib.load()
    B, N = fs.shape[0], fs.shape[1]
    ws_bytes = lib.mk_op_sample_workspace_bytes(B, IM)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)
    idx = torch.full((B * IM, N_S), -1, dtype=torch.int32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check(lib.mk_op_sample(_lib.ptr(fs), B, N, pitch, IM, N_S, seed, _lib.ptr(ws), ws_bytes, _lib.ptr(idx),
                                _lib.ptr(status), stream()))
    torch.cuda.synchronize()
    return idx.long().reshape(B, IM, N_S), int(status.item())


def test_layouts_of_the_production_matrix(prod):
    """The production matrix at its own pitch, contiguous and at pitch N + 1 (scalar loads): the same draw, which is
    the race."""
    Bq = min(prod.B, 2)
    N = prod.N
    fs = prod.fs[:Bq].contiguous()
    odd = torch.full((Bq, N, N + 1), 7.0, device=DEV)
    odd[:, :, :N] = fs
    IM = 16
    a, st_a = _sample(prod.fs[:Bq], prod.fs.stride(1), IM, 99)
    b, st_b = _sample(fs, N, IM, 99)
    c, st_c = _sample(odd, N + 1, IM, 99)
    assert st_a == st_b == st_c == 0
    assert torch.equal(a, b) and torch.equal(a, c)
    for q in range(Bq):
        stages.band_all(fs[q], b[q], q, IM, 99, f"{prod.name} layouts")


@pytest.mark.parametrize("N,IM", [(2500, 9),        # ROW_VEC with one row per 4096-cell chunk; a partial Philox group
                                  (4100, 8),        # rows longer than a chunk: scalar loads
                                  (1937, 8)])       # contiguous with N^2 odd: scalar loads
def test_sizes(N, IM):
    g = torch.Generator(device=DEV).manual_seed(N)
    p = torch.rand(1, N, N, generator=g, device=DEV) ** 8
    p[p < 1e-3] = 0
    pitch = N if N % 2 else N + 4                                       # padded rows (4-float aligned) or contiguous
    buf = torch.full((1, N, pitch), 3.0, device=DEV)
    buf[:, :, :N] = p
    idx, st = _sample(buf, pitch, IM, 1234)
    assert st == 0
    d, n = stages.band_all(p[0], idx[0], 0, IM, 1234, f"N={N}")
    print(f"\n[N={N}] max cells differing {d}, in band {n}")


def _edge(kind, g):
    N = 2500 if kind == "last_row" else 100
    p = torch.zeros(N * N, device=DEV)
    if kind.startswith("count"):
        k = int(kind[5:])
        p[torch.randperm(N * N, generator=g, device=DEV)[:k]] = torch.rand(k, generator=g, device=DEV) + 1e-3
    elif kind == "last_row":
        p[(N - 1) * N:] = torch.rand(N, generator=g, device=DEV) + 1e-3
    elif kind == "equal":
        p[torch.randperm(N * N, generator=g, device=DEV)[:6000]] = 0.25
    return p.reshape(1, N, N)


@pytest.mark.parametrize("kind", ["count2048", "count2049", "count2426", "count2427", "last_row", "equal"])
def test_edge_distributions(kind):
    """Positive counts around n_s and around the switch into all-candidates mode (target = 2048 + 8 sqrt(2048) + 16
    = 2426.04), all positives in the last row, many equal p."""
    p = _edge(kind, torch.Generator(device=DEV).manual_seed(7))
    idx, st = _sample(p, p.shape[-1], 16, 4321)
    assert st == 0
    d, n = stages.band_all(p[0], idx[0], 0, 16, 4321, kind)
    if kind == "count2048":
        assert d == 0
    print(f"\n[{kind}] max cells differing {d}, in band {n}")


@pytest.mark.parametrize("case", sorted(draws.CONTRACT))
def test_failure_contract(case):
    """The table decided by torch.multinomial (test_draws_host.py): zero pose for the whole batch exactly where it
    raises.  Pairs with fewer than 2048 positive cells draw every positive cell plus the lowest zero cells."""
    cfg, model = _model("vits", 2, 8)
    N, B, P = draws.CONTRACT_N, draws.CONTRACT_B, draws.CONTRACT_PAIR
    model._engine()._ws_for(B, 14 * 8, 14 * 8)
    fs = draws.contract_matrix(case)
    kps0, d0, kps1, d1, K = draws.contract_geometry()
    batch = {k: v.to(DEV) for k, v in dict(final_scores=fs, kps0=kps0, kps1=kps1, depth_kp0=d0, depth_kp1=d1,
                                            K_color0=K, K_color1=K).items()}
    R, t, inl = model.e2e_Procrustes.estimate_pose_vectorized(batch, seed=SEED)
    res = batch["_solver"]
    torch.cuda.synchronize()
    status = int(res["status"].item())
    zero = float(R.abs().max()) == 0 and float(t.abs().max()) == 0 and float(inl.abs().max()) == 0
    assert ("zero" if zero else "pose") == draws.CONTRACT[case], (case, status)
    assert bool(status & 1) == (draws.CONTRACT[case] == "zero") and not (status & 2)
    if zero:
        return
    assert bool(torch.isfinite(R).all()) and bool(torch.isfinite(t).all())
    got = res["sampled_idx"].long().reshape(B, 2, N_S)
    fsd = fs.to(DEV)
    for b in range(B):
        pb = fsd[b].reshape(-1)
        n_pos = int((pb > 0).sum())
        if n_pos < N_S:
            want = draws.fill_draw(pb, N_S)
            assert all(torch.equal(got[b, s], want) for s in range(2)), (case, b)
        elif case == "subnormal" and b == P:        # keys of subnormal p carry fewer bits than the band allows
            assert all(bool((pb[got[b, s]] > 0).all()) and got[b, s].unique().numel() == N_S for s in range(2))
        else:
            stages.band_all(fsd[b], got[b], b, 2, SEED, case)
    if case == "pos1":                              # ATen's fast path does not raise on CUDA either
        torch.multinomial(fsd[P].reshape(1, -1), N_S)


# ---------------------------------------------------------------------------------------------------------------
# the inner law
# ---------------------------------------------------------------------------------------------------------------
LAW_POS = [0, 7, 8, 31, 32, 255, 256, 1023, 1024, 2047]       # thread, warp and half-set seams of the cdf
LAW_W = [1.0, 0.4, 0.2, 0.1, 0.08, 0.05, 0.03, 0.01, 0.005, 0.001]


def test_inner_law():
    """X = 0 (zero depth0): every hypothesis has R = I and t = the mean of its three Y, so it decodes to its triple by
    the nearest of the C(10, 3) fp64 means.  The outer set is injected (cells 0 .. 2047 of row 0) and the inner draw
    is the kernel's.  Every triple must hold positive entries only, equal the bit-exact restatement, and follow the
    closed-form law (chi^2 p > 1e-6); the with-replacement law must be rejected."""
    B, IM, IR = 2, 16, 16384
    gh, gw = 64, 32
    N = gh * gw
    cfg, model = _model("vits", IM, IR)
    model._engine()._ws_for(B, 14 * gh, 14 * gw)
    g = torch.Generator().manual_seed(4)
    fs = torch.zeros(B, N, N)
    fs[:, 0, LAW_POS] = torch.tensor(LAW_W)
    kps0 = torch.rand(B, 2, N, generator=g) * 400
    kps1 = torch.rand(B, 2, N, generator=g) * 400
    d0 = torch.zeros(B, 1, N)
    d1 = torch.rand(B, 1, N, generator=g) * 2 + 1
    K = torch.tensor([[[300.0, 0, 224], [0, 300.0, 448], [0, 0, 1]]]).repeat(B, 1, 1)
    outer = torch.arange(N_S).repeat(B * IM, 1)
    batch = {k: v.to(DEV) for k, v in dict(final_scores=fs, kps0=kps0, kps1=kps1, depth_kp0=d0, depth_kp1=d1,
                                            K_color0=K, K_color1=K).items()}
    model.e2e_Procrustes.estimate_pose_vectorized(batch, outer_idx=outer.int(), seed=SEED)
    torch.cuda.synchronize()
    assert int(batch["_solver"]["status"].item()) == 0
    Rt = model._engine().ws_view("hyp_Rt", torch.float32, (B * IM * IR, 12)).double()
    assert float((Rt[:, :9] - torch.eye(3, device=DEV, dtype=torch.float64).reshape(1, 9)).abs().max()) == 0
    # decode: the nearest fp64 mean of a positive triple
    Y = mo.backproject(kps1.double().transpose(1, 2), d1.double().transpose(1, 2), K.double())   # [B, N, 3]
    tris = list(draws.law3(LAW_W))                                           # index triples into LAW_POS
    tri_cells = torch.tensor([[LAW_POS[i] for i in tr] for tr in tris])
    means = Y[:, tri_cells].mean(2).to(DEV)                                  # [B, 120, 3]
    sep = torch.cdist(means, means) + 1e9 * torch.eye(len(tris), device=DEV, dtype=torch.float64)
    assert float(sep.min()) > 1e-3
    t = Rt[:, 9:].reshape(B, IM * IR, 3)
    dist = torch.cdist(t, means)
    best = dist.argmin(2)
    assert float(dist.min(2).values.max()) < 1e-4                           # no triple with a zero-weight entry
    # bit-exact restatement
    w = fs[:, 0, :N_S].repeat_interleave(IM, 0).to(DEV)
    b_of = torch.arange(B, device=DEV).repeat_interleave(IM)
    idx, amb = draws.inner_draw(draws.inner_cdf(w), SEED, b_of, torch.arange(IM, device=DEV).repeat(B), IR)
    restated = idx.sort(2).values.reshape(B, IM * IR, 3)
    decoded = tri_cells.to(DEV)[best]
    mismatch = (restated != decoded).any(2) & ~amb.reshape(B, IM * IR)
    assert int(mismatch.sum()) == 0, int(mismatch.sum())
    # the law
    cnt = torch.bincount(best.reshape(-1), minlength=len(tris)).tolist()
    counts = {tris[i]: c for i, c in enumerate(cnt) if c}
    p_law = draws.chi2_pvalue(counts, draws.law3(LAW_W))
    p_repl = draws.chi2_pvalue(counts, draws.law3_with_replacement(LAW_W))
    print(f"\n[inner law] {B * IM * IR} hypotheses, {int(amb.sum())} ambiguous, chi^2 p = {p_law:.3g} "
          f"(with-replacement law: p = {p_repl:.3g})")
    assert p_law > 1e-6
    assert p_repl < 1e-6
