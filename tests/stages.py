"""The stage harness: one `compute_matches` call at any geometry, and every kernel stage of it checked element by element
against fp64 (tests/test_gpu_stages_at_scale.py at 720x540, tests/test_gpu_stages_geometries.py at other image sizes).

After the call, every intermediate whose inputs survive in the workspace (`Engine.ws_view`) is recomputed on the GPU in
fp64 from those actual inputs and the packed weights (`Engine.packed`), in chunks of images or rows, and compared with
`tests/elementwise.check`: every element within a bound derived from the arithmetic, every planted mutation of the
reference rejected.  GEMMs whose inputs the workspace overwrites later in the call are relaunched through `mk_op_gemm`
on the workspace's operands with the production parameters (engine.cu run_extract), into fresh outputs with sentinels.

Mutations sit at indices chosen from the geometry (a late M-tile, the last row of the first query tile, an interior
token), so that each one exists at every image size; each stage counts the mutations its checks rejected and `rec`
asserts that there was at least one.  `max(err / bound)` per stage goes to $MICKEY_STAGE_METRICS (a JSON file) when set.

The second half restates the solver's draws on a run (`Solved`): the outer draw against the fp64 race, the inner
triples bit for bit, each hypothesis's pose and score against fp64.
"""
import math

import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.engine import nn_pitch
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from oracle import mickey_oracle as mo
from tests import draws
from tests import elementwise as ew
from tests.common import rotation_angle_deg, synthetic_pair
from tests.gpu_util import gemm, stream

DEV = "cuda"
U32 = ew.U32
G = 4
N_S = 2048
SEED = 0x5EED5EED12345677
STAGES_WITHOUT_MUTATIONS = {"nrm2"}      # ss / (ss + 1e-10) rounds to 1 for every token: no mis-indexing changes it

# Image geometries other than 720x540 (tests/test_gpu_stages_geometries.py; tables checked on the CPU by
# tests/test_geometry_host.py): id -> (variant, B, H, W, IM, IR, GEMM regime of the relaunches), and what the geometry
# makes of the paths: (gh, gw), N, N x N row pitch, the sampler's load mode on the engine's final_scores.
GEOMETRIES = {
    "land": ("vitb", 8, 540, 720, 16, 64, "persistent"),   # landscape at the production N
    "n1920": ("vits", 1, 560, 672, 8, 64, "one tile"),    # N % 128 == 0: npad = N, pitch = N
    "t2304": ("vits", 1, 658, 686, 8, 64, "one tile"),    # T = 12 * 192 = 18 * 128, M = 36 * 128
    "crop": ("vits", 1, 727, 545, 8, 64, "one tile"),     # 13-pixel crop margins
    "min": ("vits", 1, 98, 98, 8, 64, "one tile"),        # the smallest image accepted: one interior score cell
    "sq37": ("vits", 1, 518, 518, 8, 64, "one tile"),     # 37 x 37: the position embedding as it is
    "large": ("vits", 1, 1008, 812, 8, 64, "one tile"),   # N > 4096: scalar sampler loads, no mutual matches
}
GEOMETRY_PATHS = {
    "land": ((38, 51), 1938, 1952, "ROW_VEC"),
    "n1920": ((40, 48), 1920, 1920, "FLAT_VEC"),
    "t2304": ((47, 49), 2303, 2304, "ROW_VEC"),
    "crop": ((51, 38), 1938, 1952, "ROW_VEC"),
    "min": ((7, 7), 49, 64, "ROW_VEC"),
    "sq37": ((37, 37), 1369, 1376, "ROW_VEC"),
    "large": ((72, 58), 4176, 4192, "SCALAR"),
}
SAMP_ELEMS_PER_BLOCK = 256 * 16                      # ransac.cu: cells per sampler block chunk


def sampler_mode(N, pitch, aligned=True):
    """The outer sampler's load mode for an [N, N] matrix with row pitch `pitch` floats (ransac.cu sample_outer)."""
    spr = (N + 3) // 4
    rpc = (SAMP_ELEMS_PER_BLOCK // 4) // spr
    if pitch == N and (N * N) % 4 == 0 and aligned:
        return "FLAT_VEC"
    if pitch % 4 == 0 and pitch >= 4 * spr and aligned and rpc >= 1:
        return "ROW_VEC"
    return "SCALAR"


def apply_overrides(cfg, overrides):
    """overrides: {dotted config key: value}, e.g. {'MICKEY.KP_HEADS.USE_SOFTMAX': False}; every key must exist."""
    for key, value in (overrides or {}).items():
        node = cfg
        *path, leaf = key.split(".")
        for p in path:
            node = node[p]
        assert leaf in node, key
        node[leaf] = value
    return cfg


class Run:
    """One compute_matches call on B synthetic pairs of H x W images and the geometry of its workspace.  A crop margin
    (H or W not a multiple of 14) is filled with NaN: the patch gather must never read it.  `overrides` changes the
    configuration of mickey_cfg (apply_overrides): the head and matcher flags the stage checks follow."""

    def __init__(self, name, variant, B, H, W, im, ir, regime=None, overrides=None):
        self.name, self.B, self.H, self.W, self.im, self.ir = name, B, H, W, im, ir
        self.regime = regime                     # "persistent" / "one tile" / None: what the relaunched GEMMs must use
        self.cfg = apply_overrides(mickey_cfg(variant, im, ir), overrides)
        m = self.cfg.MICKEY
        self.use_softmax, self.depth_sigmoid = bool(m.KP_HEADS.USE_SOFTMAX), bool(m.KP_HEADS.USE_DEPTHSIGMOID)
        self.max_depth, self.norm_dsc = float(m.KP_HEADS.MAX_DEPTH), bool(m.DSC_HEAD.NORM_DSC)
        self.use_dustbin = bool(self.cfg.FEATURE_MATCHER.DUAL_SOFTMAX.USE_DUSTBIN)
        self.temperature = float(self.cfg.FEATURE_MATCHER.DUAL_SOFTMAX.TEMPERATURE)
        model = MickeyRelativePose(self.cfg)
        model.load_state_dict(synthetic_state_dict(self.cfg, seed=3), strict=True)
        self.model = model.cuda().eval()
        self.gh, self.gw = H // 14, W // 14
        pair = synthetic_pair(B, H, W, seed=17)
        for k in ("image0", "image1"):
            pair[k][:, :, 14 * self.gh:] = float("nan")
            pair[k][:, :, :, 14 * self.gw:] = float("nan")
        self.data = {k: v.to(DEV) for k, v in pair.items()}
        with torch.no_grad():
            self.model.compute_matches(self.data)
        torch.cuda.synchronize()
        self.eng = self.model._engine()
        c = self.eng.mkcfg
        self.D, self.heads, self.depth, self.bd = c.embed_dim, c.heads, c.depth, list(c.block_dims)
        self.n_img = 2 * B
        self.N = self.gh * self.gw
        self.T = self.N + 1
        self.h2, self.w2 = self.gh + 2, self.gw + 2
        self.per_img = self.h2 * self.w2
        self.R, self.M, self.Mp = self.n_img * self.per_img, self.n_img * self.T, self.n_img * self.N
        self.npad = -(-self.N // 128) * 128
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        pos = torch.arange(self.per_img, device=DEV)
        y, x = pos // self.w2, pos % self.w2
        self.valid_pos = (y >= 1) & (y <= self.h2 - 2) & (x >= 1) & (x <= self.w2 - 2)
        self.valid = self.valid_pos.repeat(self.n_img)                 # [R]
        self.images = torch.cat([self.data["image0"], self.data["image1"]], 0)
        self.interior = 3 * self.gw + 3                                 # first token inside the score map's 3-cell border
        self.rejected = {}

    def ws(self, name, dtype, *shape):
        return self.eng.ws_view(name, dtype, shape)

    def w(self, name):
        return self.eng.packed[name]

    def rows(self, kind):
        return {"padded": ew.Rows("padded", self.per_img, self.w2), "tokens": ew.Rows("tokens", self.T),
                "patches": ew.Rows("patches", self.N)}[kind]

    def tiles(self, M, N, groups=1, group_fast=False):
        return ew.GemmTiles(M, N, groups, group_fast, self.sms)

    def valid_pair(self, p):
        """The first padded position >= p of an image whose right neighbour is also a valid position."""
        v = self.valid_pos
        while not (bool(v[p]) and bool(v[p + 1])):
            p += 1
        return p


def check(run, stage, name, got, ref, bound, where=None, mutations=()):
    r = ew.check(name, got, ref, bound, where, mutations)
    run.rejected[stage] = run.rejected.get(stage, 0) + len(mutations)
    return r


def check_exact(run, stage, name, got, ref, where=None, mutations=()):
    ew.check_exact(name, got, ref, where, mutations)
    run.rejected[stage] = run.rejected.get(stage, 0) + len(mutations)


def rec(run, stage, ratio):
    """Record max(err / bound) of a stage; every stage must have rejected at least one planted mutation."""
    n = run.rejected.get(stage, 0)
    assert n > 0 or stage in STAGES_WITHOUT_MUTATIONS, f"{run.name} {stage}: no mutation was planted"
    print(f"\n[{run.name}] {stage}: max err/bound {ratio:.3g}, {n} planted mutations rejected", end="")
    ew.record(stage, run.name, ratio)
    return ratio


def _chunks(n, size):
    for i in range(0, n, size):
        yield i, min(n, i + size)


# ---------------------------------------------------------------------------------------------------------------
# generic GEMM-family checks (fp64 reference from the exact fp16 operands, bound from tests/elementwise.py)
# ---------------------------------------------------------------------------------------------------------------
def _shifted_slab(A, col0, cin, r0, r1, halo):
    """A[r0 - halo : r1 + halo, col0 : col0 + cin] in fp64, zero outside the tensor (TMA zero fill)."""
    R = A.shape[0]
    out = torch.zeros(r1 - r0 + 2 * halo, cin, dtype=torch.float64, device=DEV)
    lo, hi = max(0, r0 - halo), min(R, r1 + halo)
    out[lo - (r0 - halo):hi - (r0 - halo)] = A[lo:hi, col0:col0 + cin].double()
    return out


def conv_ref(run, A, col0, cin, Wg, r0, r1, three):
    """Shifted-row conv (or 1x1) of rows r0..r1: (pre, |A||W|, slab, shifts, halo) in fp64."""
    shifts = [(ky - 1) * run.w2 + (kx - 1) for ky in range(3) for kx in range(3)] if three else [0]
    halo = run.w2 + 2 if three else 0
    slab = _shifted_slab(A, col0, cin, r0, r1, halo)
    n = r1 - r0
    Wd = Wg.double()
    pre = torch.zeros(n, Wg.shape[0], dtype=torch.float64, device=DEV)
    ab = torch.zeros_like(pre)
    for t, s in enumerate(shifts):
        a = slab[halo + s:halo + s + n]
        wt = Wd[:, t * cin:(t + 1) * cin]
        pre += a @ wt.t()
        ab += a.abs() @ wt.abs().t()
    return pre, ab, slab, shifts, halo


def check_conv(run, stage, A, cin, Wfull, groups, cout, three, got_of, *, a_col0, bias=None, res_of=None, act="relu",
               pe=None, pe_groups=(), pad_mask=True, fp16_out=True, group_fast=False, row_chunk=16384):
    """EPI_CONV: mask(act(conv(A_g) + bias_g + res_g) + pe) for every group g, compared with got_of(g, r0, r1)."""
    R = run.R
    tiles = run.tiles(R, cout, groups, group_fast)
    worst = 0.0
    mut_tile = max(0, R // 128 - 2)                                  # a full M-tile in the last rounds
    planted = 0
    for g in range(groups):
        Wg = Wfull[g * cout:(g + 1) * cout]
        b = bias[g * cout:(g + 1) * cout].double() if bias is not None else None
        for r0, r1 in _chunks(R, row_chunk):
            pre, ab, slab, shifts, halo = conv_ref(run, A, a_col0(g), cin, Wg, r0, r1, three)
            res = res_of(g, r0, r1).double() if res_of is not None else None
            pos = torch.arange(r0, r1, device=DEV) % run.per_img
            pe_t = pe[pos].double() if (pe is not None and g in pe_groups) else None

            def post(p, rows):
                t = p + (b if b is not None else 0) + (res[rows] if res is not None else 0)
                t = t.relu() if act == "relu" else t
                if pe_t is not None:
                    t = t + pe_t[rows]
                if pad_mask:
                    t = torch.where(run.valid[r0:r1][rows, None], t, torch.zeros_like(t))
                return t

            allr = slice(None)
            ref = post(pre, allr)
            bound = (ew.gemm_acc_bound(len(shifts) * cin, ab)
                     + ew.epilogue_terms(pre, b, res, pe_t, ref) + ew.out_rounding(ref, fp16_out))
            if pad_mask:
                bound = torch.where(run.valid[r0:r1][:, None], bound, torch.zeros_like(bound))
            bound = bound.clamp_min(1e-30)
            muts = []
            m0 = mut_tile * 128
            if g == groups - 1 and r0 <= m0 and m0 + 128 <= r1:
                rows = slice(m0 - r0, m0 - r0 + 128)
                cols = slice(0, min(cout, tiles.bn))
                kc = len(shifts) * cin // 64 - 1                     # the tile's last K chunk
                t, kin = divmod(kc, cin // 64)
                a = slab[halo + shifts[t] + m0 - r0:halo + shifts[t] + m0 - r0 + 128, kin * 64:(kin + 1) * 64]
                w = Wg[cols, t * cin + kin * 64:t * cin + (kin + 1) * 64].double()
                muts.append(ew.Mutation(f"K chunk {kc} dropped from M-tile {mut_tile}", (rows, cols),
                                        post(pre[rows] - torch.nn.functional.pad(a @ w.t(), (0, pre.shape[1] - w.shape[0])), rows)[:, cols]))
                if three:
                    mid = m0 - r0 + 64 + int(run.valid[m0 + 64:m0 + 128].nonzero()[0])     # a valid row of the tile
                    a0 = slab[halo + shifts[4] + mid:halo + shifts[4] + mid + 1]
                    a1 = slab[halo + shifts[4] + run.w2 + mid:halo + shifts[4] + run.w2 + mid + 1]
                    wt = Wg[:, 4 * cin:5 * cin].double()
                    muts.append(ew.Mutation("centre tap read one padded row off", (slice(mid, mid + 1), allr),
                                            post(pre[mid:mid + 1] - a0 @ wt.t() + a1 @ wt.t(), slice(mid, mid + 1))))
                vr = int(run.valid[r0:r1].nonzero()[len(run.valid[r0:r1].nonzero()) // 2])
                muts.append(ew.row_chunk_swap(ref, vr, 0))
                if pe_t is not None:
                    muts.append(ew.Mutation("PE row of the neighbouring position", (slice(vr, vr + 1), allr),
                                            (ref[vr:vr + 1] - pe_t[vr:vr + 1] + pe[pos[vr] + 1].double())))
            if pe is not None and g not in pe_groups and r0 == 0:
                # the PE on a group whose POS_ENCODING flag is off (a wrong aux_group_mask)
                vr = int(run.valid[r0:r1].nonzero()[0])
                muts.append(ew.Mutation(f"PE added to group {g}, whose flag is off", (slice(vr, vr + 1), allr),
                                        ref[vr:vr + 1] + pe[pos[vr]].double()))
            planted += len(muts)
            where = ew.matrix_where(run.rows("padded"), tiles, row_offset=r0)
            where_g = ew.Where(lambda idx, g=g: (int(idx[0]), g, int(idx[1])), where.rows, tiles, r0)
            worst = max(worst, check(run, stage, f"{run.name} {stage} group {g}", got_of(g, r0, r1), ref, bound, where_g, muts))
            assert not muts or g == groups - 1 or (pe is not None and g not in pe_groups)
    assert planted > 0, f"{run.name} {stage}: no mutation planted (R = {R})"
    return rec(run, stage, worst)


# ---------------------------------------------------------------------------------------------------------------
# §3: the stage chain
# ---------------------------------------------------------------------------------------------------------------
def patch_gather(run):
    P = run.ws("P", torch.float16, run.Mp, 640)
    gh, gw = run.gh, run.gw
    for i0, i1 in _chunks(run.n_img, 8):
        im = run.images[i0:i1, :, :gh * 14, :gw * 14]
        ref = im.reshape(i1 - i0, 3, gh, 14, gw, 14).permute(0, 2, 4, 1, 3, 5).reshape(-1, 588).half()
        got = P[i0 * run.N:i1 * run.N]
        muts = [ew.Mutation("token of the neighbouring image", (slice(5, 6),), ref[run.N + 5:run.N + 6])] if i1 - i0 > 1 else []
        check_exact(run, "patch_gather", f"{run.name} P", got[:, :588], ref,
                    ew.matrix_where(run.rows("patches"), row_offset=i0 * run.N), muts)
        assert float(got[:, 588:].abs().max()) == 0.0, "K-pad columns 588..639 of P are not zero"
    rec(run, "patch_gather", 0.0)


def final_layernorm_and_scatter(run):
    X = run.ws("X", torch.float32, run.n_img, run.T, run.D)
    Fm = run.ws("F", torch.float16, run.n_img, run.h2, run.w2, run.D)
    w, b = run.w("norm.w").double(), run.w("norm.b").double()
    worst = 0.0
    for i0, i1 in _chunks(run.n_img, 8):
        ref, bound = ew.ln_bound(X[i0:i1, 1:].double(), 0.0, w, b, 1e-6)
        bound = bound + ew.out_rounding(ref, True)
        got = Fm[i0:i1, 1:-1, 1:-1].reshape(i1 - i0, run.N, run.D)
        muts = [ew.Mutation("token of the neighbouring image", (0, slice(7, 8)), ref[1, 7:8]),
                ew.Mutation("32 columns of the next token", (0, slice(7, 8), slice(32, 64)), ref[0, 8:9, 32:64])] if i1 - i0 > 1 else []
        where = ew.Where(lambda idx, i0=i0: ((i0 + int(idx[0])) * run.N + int(idx[1]), 0, int(idx[2])), run.rows("patches"))
        worst = max(worst, check(run, "final_layernorm", f"{run.name} F", got, ref, bound, where, muts))
        ring = Fm[i0:i1].clone()
        ring[:, 1:-1, 1:-1] = 0
        assert float(ring.abs().max()) == 0.0, "pad ring of F is not zero"
    rec(run, "final_layernorm", worst)


def last_block_attention(run):
    D, T, nh = run.D, run.T, run.heads
    QKV = run.ws("QKV", torch.float16, run.n_img, T, 3, nh, 64)
    ATT = run.ws("ATT", torch.float16, run.n_img, T, nh, 64)
    qt = -(-T // 192)
    tiles = run.n_img * nh * qt
    grid = min(tiles, run.sms)
    assert run.name != "C3" or tiles == 8448
    q_last = min(191, T - 2)                       # the last row of the first query tile (or of the only one)

    class AttnWhere(ew.Where):
        def describe(self, idx, img=0):
            h, t, c = (int(i) for i in idx)
            tile = (self.img * nh + h) * qt + t // 192
            return (f"image {self.img}, head {h}, query {t}, dim {c}; attention tile {tile} (query tile {t // 192}), "
                    f"round {tile // grid} of {grid} persistent CTAs")

    worst = 0.0
    for img in range(run.n_img):
        q, k, v = (QKV[img, :, j].permute(1, 0, 2).double() for j in range(3))
        ref, bound = ew.attention_ref_bound(q, k, v)
        got = ATT[img].permute(1, 0, 2)
        muts = []
        if img == run.n_img - 1:
            sw = ew.row_chunk_swap(ref[0], q_last, 32)
            qn = min(200, T - 1)
            muts = [ew.Mutation(sw.label, (0,) + sw.idx, sw.values),
                    ew.Mutation("output of the next head", (0, slice(qn, qn + 1)), ref[1, qn:qn + 1])]
        wh = AttnWhere()
        wh.img = img
        worst = max(worst, check(run, "attention", f"{run.name} ATT", got, ref, bound, wh, muts))
        del ref, bound
    rec(run, "attention", worst)


def _linear_check(run, stage, A, Wt, bias, got, *, act=None, fp16_out=True, tiles=None, rows="tokens", row_chunk=8192,
                  resid=None, gamma=None, group=0):
    """out = act(A W^T + bias) (fp16 or fp32) or resid + gamma (A W^T + bias) (fp32, EPI_RESID_F), rows in chunks;
    the planted mutations go into the chunk holding row M - 256 (a late persistent round), or into M-tile 0 when M
    is smaller than that."""
    M, K = A.shape
    Wd, b = Wt.double(), bias.double()
    gm = gamma.double() if gamma is not None else None
    worst = 0.0
    mut_chunk = max(0, (M - 256) // row_chunk * row_chunk)
    planted = 0
    for r0, r1 in _chunks(M, row_chunk):
        a = A[r0:r1].double()
        pre = a @ Wd.t()
        acc_b = ew.gemm_acc_bound(K, a.abs() @ Wd.abs().t())
        x0 = resid[r0:r1].double() if resid is not None else None

        def post(p, rows=slice(None)):
            t = p + b
            if act == "gelu":
                return ew.gelu64(t)
            if act == "relu":
                return t.relu()
            if x0 is not None:
                return x0[rows] + gm * t
            return t

        ref = post(pre)
        if act == "gelu":
            bound = ew.gelu_bound(pre + b, acc_b + ew.epilogue_terms(pre, b))
        elif x0 is not None:
            bound = gm.abs() * (acc_b + ew.epilogue_terms(pre, b)) + ew.epilogue_terms(ref, x0)
        else:
            bound = acc_b + ew.epilogue_terms(pre, b)
        bound = (bound + ew.out_rounding(ref, fp16_out)).clamp_min(1e-30)
        muts = []
        if r0 == mut_chunk:
            m0 = max(0, (M - 256 - r0) // 128 * 128)              # a whole M-tile inside this chunk (clipped at M)
            tr = slice(m0, m0 + 128)
            kc = K // 64 - 1
            dropped = pre[tr].clone()
            dropped[:, :128] -= a[tr, kc * 64:(kc + 1) * 64] @ Wd[:128, kc * 64:(kc + 1) * 64].t()
            muts = [ew.Mutation(f"K chunk {kc} dropped from one tile", (tr, slice(0, 128)), post(dropped, tr)[:, :128]),
                    ew.row_chunk_swap(ref, m0 + 64, 32)]
        planted += len(muts)
        where = ew.Where(lambda idx: (int(idx[0]), group, int(idx[1])), run.rows(rows),
                         tiles, r0)
        worst = max(worst, check(run, stage, f"{run.name} {stage}", got[r0:r1], ref, bound, where, muts))
    assert planted > 0, f"{run.name} {stage}: no mutation planted (M = {M})"
    return rec(run, stage, worst)


def last_block_fc1_gelu(run):
    D, M = run.D, run.M
    blk = f"blk{run.depth - 1}."
    XN = run.ws("XN", torch.float16, M, D)
    H1 = run.ws("H1", torch.float16, M, 4 * D)
    _linear_check(run, "fc1_gelu", XN, run.w(blk + "fc1.w"), run.w(blk + "fc1.b"), H1, act="gelu",
                  tiles=run.tiles(M, 4 * D))


def head_residual_blocks(run):
    R, D, bd = run.R, run.D, run.bd
    ins = [("F", D, 0), ("O1", bd[0], bd[0]), ("O2", bd[1], bd[1])]
    for r in range(3):
        cout = bd[r]
        name_in, cin, goff = ins[r]
        A = run.ws(name_in, torch.float16, R, D if r == 0 else G * cin)
        Tt = run.ws(f"T{r + 1}", torch.float16, R, G * cout)
        S = run.ws(f"S{r + 1}", torch.float16, R, G * cout)
        n = f"rb{r + 1}."
        gsl = lambda t, g, r0, r1, c=cout: t[r0:r1, g * c:(g + 1) * c]        # noqa: E731
        check_conv(run, f"rb{r + 1}.conv1", A, cin, run.w(n + "c1.w"), G, cout, True, lambda g, r0, r1: gsl(Tt, g, r0, r1),
                   a_col0=lambda g, goff=goff: g * goff, bias=run.w(n + "c1.b"), group_fast=(r == 0))
        check_conv(run, f"rb{r + 1}.shortcut", A, cin, run.w(n + "sc.w"), G, cout, False, lambda g, r0, r1: gsl(S, g, r0, r1),
                   a_col0=lambda g, goff=goff: g * goff, act="none", pad_mask=False, group_fast=(r == 0))
        if r < 2:
            O = run.ws(f"O{r + 1}", torch.float16, R, G * cout)
            check_conv(run, f"rb{r + 1}.conv2", Tt, cout, run.w(n + "c2.w"), G, cout, True, lambda g, r0, r1: gsl(O, g, r0, r1),
                       a_col0=lambda g: g * cout, bias=run.w(n + "c2.b"), res_of=lambda g, r0, r1: gsl(S, g, r0, r1))


def _elu1(x):
    return torch.where(x > 0, x + 1.0, torch.exp(x))


def linear_attention_last_layer(run):
    n_img, L = run.n_img, run.N
    QKV32 = run.ws("QKV32", torch.float32, n_img, run.per_img, G, 3, 8, 16)
    KV = run.ws("KV", torch.float32, n_img, G, 8, 272)
    MSG = run.ws("MSG", torch.float16, n_img, run.per_img, G, 8, 16)
    vp = run.valid_pos
    pm = run.valid_pair(min(100, run.per_img // 2))     # a valid position whose right neighbour is valid
    w_kv = w_msg = w_msg64 = 0.0
    for i0, i1 in _chunks(n_img, 8):
        q = QKV32[i0:i1].double()
        Kf = _elu1(q[:, vp, :, 1])                       # [n, L, G, 8, 16]
        V = q[:, vp, :, 2] / L
        kv = torch.einsum("nsghd,nsghv->nghdv", Kf, V)
        kv_abs = torch.einsum("nsghd,nsghv->nghdv", Kf, V.abs())
        ks = Kf.sum(1)                                   # [n, G, 8, 16]
        ref = torch.cat([kv.reshape(i1 - i0, G, 8, 256), ks], -1)
        bnd = torch.cat([kv_abs.reshape(i1 - i0, G, 8, 256), ks], -1) * (L + 6) * U32
        got = KV[i0:i1]
        muts = [ew.Mutation("KV of the neighbouring image", (0,), ref[1])] if i1 - i0 > 1 else []
        muts.append(ew.Mutation("Ksum of the next head", (0, 0, 0, slice(256, 272)), ref[0, 0, 1, 256:272]))
        w_kv = max(w_kv, check(run, "linattn_kv", f"{run.name} KV", got, ref, bnd.clamp_min(1e-30), mutations=muts))
        # MSG from the kernel's own KV (isolates the message kernel), then from the fp64 KV (the pair of kernels)
        Q = _elu1(q[:, :, :, 0])                         # [n, P, G, 8, 16]
        for kvsrc, kvb, tag, stage in ((got.double(), None, "MSG", "linattn_msg"),
                                       (ref, bnd, "MSG_vs_fp64_KV", "linattn_msg_vs_fp64_kv")):
            kvm, ksm = kvsrc[..., :256].reshape(i1 - i0, G, 8, 16, 16), kvsrc[..., 256:]
            num = torch.einsum("npghd,nghdv->npghv", Q, kvm)
            num_abs = torch.einsum("npghd,nghdv->npghv", Q, kvm.abs())
            den = torch.einsum("npghd,nghd->npgh", Q, ksm)[..., None] + 1e-6
            den_b = (20 * U32 + 2.0 ** -22) * (den - 1e-6)
            num_b = (20 * U32 + 2.0 ** -22) * num_abs
            if kvb is not None:
                kb = kvb[..., :256].reshape(i1 - i0, G, 8, 16, 16)
                num_b = num_b + torch.einsum("npghd,nghdv->npghv", Q, kb)
                den_b = den_b + torch.einsum("npghd,nghd->npgh", Q, kvb[..., 256:])[..., None]
            z = L / den
            m_ref = num * z
            m_b = z * num_b + m_ref.abs() * (den_b / den + 3 * U32) + ew.out_rounding(m_ref, True)
            gm = MSG[i0:i1]
            muts = [ew.Mutation("message of the next position", (0, slice(pm, pm + 1)), m_ref[0, pm + 1:pm + 2]),
                    ew.Mutation("message of the neighbouring group", (0, slice(pm, pm + 1), 0), m_ref[0, pm:pm + 1, 1])]
            r = check(run, stage, f"{run.name} {tag}", gm, m_ref, m_b, mutations=muts)
            if tag == "MSG":
                w_msg = max(w_msg, r)
            else:
                w_msg64 = max(w_msg64, r)
    rec(run, "linattn_kv", w_kv)
    rec(run, "linattn_msg", w_msg)
    rec(run, "linattn_msg_vs_fp64_kv", w_msg64)


def head_transformer_outputs(run):
    """CAT[:, g*256+128:] = LN(MSG_g W_merge^T) gamma + beta on valid rows (EPI_LN without a residual);
    CAT[:, g*256:+128] = fp16(X32_g) exactly, both zero on pad rows (mlp2_ln with pad zeroing)."""
    R = run.R
    CAT = run.ws("CAT", torch.float16, R, G, 256)
    MSG = run.ws("MSG", torch.float16, R, G, 128)
    X32 = run.ws("X32", torch.float32, R, G, 128)
    Wm, n1w, n1b = run.w("att2.merge.w"), run.w("att2.n1.w"), run.w("att2.n1.b")
    worst = 0.0
    vidx = run.valid.nonzero()[:, 0]
    for g in range(G):
        Wg = Wm[g * 128:(g + 1) * 128].double()
        for c0, c1 in _chunks(vidx.numel(), 32768):
            rows = vidx[c0:c1]
            a = MSG[rows, g].double()
            acc = a @ Wg.t()
            e = ew.gemm_acc_bound(128, a.abs() @ Wg.abs().t())
            ref, b = ew.ln_bound(acc, e, n1w[g * 128:(g + 1) * 128].double(), n1b[g * 128:(g + 1) * 128].double(), 1e-5)
            b = b + ew.out_rounding(ref, True)
            muts = [ew.row_chunk_swap(ref, 10, 96)] if g == G - 1 and c0 == 0 else []
            where = ew.Where(lambda idx, rows=rows, g=g: (int(rows[int(idx[0])]), g, 128 + int(idx[1])), run.rows("padded"))
            worst = max(worst, check(run, "merge_ln", f"{run.name} CAT merge_ln", CAT[rows, g, 128:], ref, b, where, muts))
    rec(run, "merge_ln", worst)
    x16 = X32.half()
    check_exact(run, "mlp2_ln_cat_copy", f"{run.name} CAT = fp16(X32)", CAT[:, :, :128], x16,
                ew.Where(lambda idx: (int(idx[0]), int(idx[1]), int(idx[2])), run.rows("padded")),
                [ew.Mutation("group 0 copied from group 1", (slice(None), 0), x16[:, 1])])
    pad = ~run.valid
    assert float(X32[pad].abs().max()) == 0.0 and float(CAT[pad][:, :, :128].abs().max()) == 0.0
    rec(run, "mlp2_ln_cat_copy", 0.0)


def block4(run):
    R = run.R
    CAT = run.ws("CAT", torch.float16, R, G * 256)
    co = run.bd[3]
    T4k, S4k = run.ws("T4k", torch.float16, R, 3 * co), run.ws("S4k", torch.float16, R, 3 * co)
    Y4k = run.ws("Y4k", torch.float32, R, 3 * co)
    gs = lambda t, g, r0, r1, c=co: t[r0:r1, g * c:(g + 1) * c]               # noqa: E731
    check_conv(run, "rb4k.conv1", CAT, 128, run.w("rb4k.c1.w"), 3, co, True, lambda g, r0, r1: gs(T4k, g, r0, r1),
               a_col0=lambda g: g * 256, bias=run.w("rb4k.c1.b"))
    check_conv(run, "rb4k.shortcut", CAT, 128, run.w("rb4k.sc.w"), 3, co, False, lambda g, r0, r1: gs(S4k, g, r0, r1),
               a_col0=lambda g: g * 256, act="none", pad_mask=False)
    check_conv(run, "rb4k.conv2", T4k, co, run.w("rb4k.c2.w"), 3, co, True, lambda g, r0, r1: gs(Y4k, g, r0, r1),
               a_col0=lambda g: g * co, bias=run.w("rb4k.c2.b"), res_of=lambda g, r0, r1: gs(S4k, g, r0, r1), fp16_out=False)
    T4d, Y4d = run.ws("T4d", torch.float16, R, 128), run.ws("Y4d", torch.float32, R, 128)
    check_conv(run, "rb4d.conv1", CAT, 128, run.w("rb4d.c1.w"), 1, 128, True, lambda g, r0, r1: T4d[r0:r1],
               a_col0=lambda g: 768, bias=run.w("rb4d.c1.b"))
    check_conv(run, "rb4d.conv2", T4d, 128, run.w("rb4d.c2.w"), 1, 128, True, lambda g, r0, r1: Y4d[r0:r1],
               a_col0=lambda g: 0, bias=run.w("rb4d.c2.b"), res_of=lambda g, r0, r1: CAT[r0:r1, 768:896], act="none",
               fp16_out=False)


def head_outputs(run):
    n_img, N, B = run.n_img, run.N, run.B
    vidx = run.valid.nonzero()[:, 0]
    Y4k = run.ws("Y4k", torch.float32, run.R, 192)[vidx].double().reshape(n_img, N, 192)
    Y4d = run.ws("Y4d", torch.float32, run.R, 128)[vidx].double().reshape(n_img, N, 128)
    d = run.data
    wd, wxy, ws_ = run.w("out.depth.w").double(), run.w("out.xy.w").double(), run.w("out.score.w").double()

    def dot(y, w):
        return y @ w, (64 + 2) * U32 * (y.abs() @ w.abs())

    a_d, b_d = dot(Y4k[..., :64], wd)
    a_x, b_x = dot(Y4k[..., 64:128], wxy[:64])
    a_y, b_y = dot(Y4k[..., 64:128], wxy[64:])
    a_s, b_s = dot(Y4k[..., 128:], ws_)
    depth = torch.cat([d["depth_kp0"], d["depth_kp1"]], 0)[:, 0]
    kps = torch.cat([d["kps0"], d["kps1"]], 0)
    score_raw = run.ws("score_raw", torch.float32, n_img, N)
    if run.depth_sigmoid:
        # MAX_DEPTH sigma(a): the dot's error through sigma' <= sigma (1 - sigma); one expf (2 ulp), one add, one division
        sg = torch.sigmoid(a_d)
        d_ref = run.max_depth * sg
        d_b = run.max_depth * sg * (1 - sg) * b_d + 8 * U32 * d_ref.abs() + 1e-37
        muts = [ew.Mutation("token of the neighbouring image", (0, slice(9, 10)), d_ref[1, 9:10]),
                ew.Mutation("MAX_DEPTH dropped from the depth sigmoid", (0, slice(9, 10)), sg[0, 9:10])]
    else:
        d_ref, d_b = a_d, b_d + U32 * a_d.abs()
        muts = [ew.Mutation("token of the neighbouring image", (0, slice(9, 10)), a_d[1, 9:10])]
    rec(run, "depth", check(run, "depth", f"{run.name} depth", depth, d_ref, d_b.clamp_min(1e-30), mutations=muts))
    rec(run, "score_raw", check(run, "score_raw", f"{run.name} score_raw", score_raw, a_s,
                                (b_s + U32 * a_s.abs()).clamp_min(1e-30),
                                mutations=[ew.Mutation("next token", (0, slice(9, 10)), a_s[0, 10:11])]))
    n = torch.arange(N, device=DEV)
    xx, yy = (n % run.gw).double(), (n // run.gw).double()
    ref_k = torch.stack([(torch.sigmoid(a_x) + xx) * 14, (torch.sigmoid(a_y) + yy) * 14], 1)
    bk = torch.stack([14 * (0.25 * b_x + 2.0 ** -22 + 3 * U32), 14 * (0.25 * b_y + 2.0 ** -22 + 3 * U32)], 1) + 2 * U32 * ref_k.abs()
    kt = 50 if N > 50 else 1                         # a token whose grid x and y differ
    rec(run, "kps", check(run, "kps", f"{run.name} kps", kps, ref_k, bk,
                          mutations=[ew.Mutation("x and y swapped", (0, slice(0, 1), slice(kt, kt + 1)),
                                                 ref_k[0, 1:2, kt:kt + 1])]))
    r = score_raw.double()
    inside = ((yy >= 3) & (yy < run.gh - 3) & (xx >= 3) & (xx < run.gw - 3))
    scr = torch.cat([d["scr0"], d["scr1"]], 0)[:, 0]
    c = int(inside.nonzero()[0])
    assert c == run.interior
    if run.use_softmax:
        # score activation: spatial softmax (temperature 100) of the kernel's own raw map, 3-pixel border exactly zero
        mean = r.mean(-1, keepdim=True) + 1e-16
        arg = (r - mean) / 100
        e = torch.where(inside, torch.exp(arg), torch.zeros_like(arg))
        scr_ref = e / (e.sum(-1, keepdim=True) + 1e-16)
        d_arg = (N * U32 * r.abs().mean(-1, keepdim=True) + U32 * mean.abs()) / 100 + 2 * U32 * arg.abs()
        rel = 2 * (d_arg.amax(-1, keepdim=True) + 2.0 ** -22) + (N + 2) * U32
        bnd = torch.where(inside, scr_ref * rel, torch.zeros_like(scr_ref)).clamp_min(1e-30)
        rec(run, "score_softmax", check(run, "score_softmax", f"{run.name} scr", scr, scr_ref, bnd,
                                        mutations=[ew.Mutation("next token", (0, slice(c, c + 1)), scr_ref[0, c + 1:c + 2])]))
        assert float((scr.double().sum(-1) - 1).abs().max()) <= float(rel.max()) + N * U32
    else:
        # sigmoid(raw) inside the 3-cell border, exactly 0 outside: one expf (2 ulp) and one division of the kernel's own
        # raw map (an expf that overflows gives 0 where sigmoid < 1e-37)
        sg = torch.sigmoid(r)
        scr_ref = torch.where(inside, sg, torch.zeros_like(sg))
        bnd = torch.where(inside, 8 * U32 * scr_ref + 1e-37, torch.zeros_like(scr_ref)).clamp_min(1e-30)
        rec(run, "score_sigmoid", check(run, "score_sigmoid", f"{run.name} scr", scr, scr_ref, bnd, mutations=[
            ew.Mutation("next token", (0, slice(c, c + 1)), scr_ref[0, c + 1:c + 2]),
            ew.Mutation("border dropped from the sigmoid score", (0, slice(0, 1)), sg[0, 0:1])]))
    # descriptors: d / sqrt(sum d^2 + 1e-10) (or d itself without DSC_HEAD.NORM_DSC), the squared norm of what is stored,
    # and the split operand of the matcher (bit-exact)
    ss = (Y4d * Y4d).sum(-1, keepdim=True)
    normed = Y4d / torch.sqrt(ss + 1e-10)
    dsc = torch.cat([d["dsc0"], d["dsc1"]], 0).transpose(1, 2)
    nrm2 = run.ws("nrm2", torch.float32, n_img, N)
    if run.norm_dsc:
        rel_d = (129 / 2 + 4) * U32
        rec(run, "dsc", check(run, "dsc", f"{run.name} dsc", dsc, normed, (normed.abs() * rel_d).clamp_min(1e-30),
                              mutations=[ew.Mutation("channels of the next token", (0, slice(3, 4)), normed[0, 4:5])]))
        n2_ref = ss[..., 0] / (ss[..., 0] + 1e-10)
        rec(run, "nrm2", check(run, "nrm2", f"{run.name} nrm2", nrm2, n2_ref, (129 + 2 * 69 + 4) * U32 * n2_ref.abs() + 1e-30))
    else:
        # desc_out_kernel stores Y4d as it is and its fp32 sum of squares (4 per lane, then a 5-step butterfly)
        y32 = Y4d.float()
        check_exact(run, "dsc", f"{run.name} dsc = Y4d", dsc, y32,
                    mutations=[ew.Mutation("channels of the next token", (0, slice(3, 4)), y32[0, 4:5]),
                               ew.Mutation("normalisation applied without NORM_DSC", (0, slice(3, 4)), normed[0, 3:4].float())])
        rec(run, "dsc", 0.0)
        n2_ref = ss[..., 0]
        rec(run, "nrm2", check(run, "nrm2", f"{run.name} nrm2", nrm2, n2_ref, (129 * U32 * n2_ref).clamp_min(1e-30),
                               mutations=[ew.Mutation("normalisation applied without NORM_DSC", (0, slice(3, 4)),
                                                      (ss[0, 3:4, 0] / (ss[0, 3:4, 0] + 1e-10)))]))
    DSCX = run.ws("DSCX", torch.float16, n_img, N, 384)
    hi, lo = ew.split_hi_lo(dsc.contiguous())
    ref_x = torch.cat([torch.cat([hi[:B], lo[:B], hi[:B]], -1), torch.cat([hi[B:], hi[B:], lo[B:]], -1)], 0)
    swapped = torch.cat([lo[:1], hi[:1], hi[:1]], -1)
    check_exact(run, "dscx", f"{run.name} DSCX", DSCX, ref_x,
                mutations=[ew.Mutation("hi and lo swapped in role 0", (slice(0, 1),), swapped)])
    rec(run, "dscx", 0.0)


def _resolvable(v, bound, i=40):
    """i when v[i + 1] differs from v[i] by more than twice i's bound, else the index where that margin is largest."""
    if float((v[i + 1] - v[i]).abs()) > 2 * float(bound[i]):
        return i
    return int(((v[1:] - v[:-1]).abs() - 2 * bound[:-1]).argmax())


def _swap_at(ref, bound, r, c):
    """(r, c) when columns c..c+31 of row r + 1 differ from row r's by more than twice the bound somewhere, else the
    row and 32-column chunk where that margin is largest (scores concentrated on a few cells at T = 1)."""
    margin = (ref[:-1] - ref[1:]).abs() - 2 * bound[:-1]
    if float(margin[r, c:c + 32].max()) > 0:
        return r, c
    i = int(margin.argmax())
    return i // ref.shape[1], max(0, min(i % ref.shape[1] - 16, ref.shape[1] - 32))


def matcher(run):
    B, N, npad = run.B, run.N, run.npad
    DSCX = run.ws("DSCX", torch.float16, run.n_img, N, 384)
    lse_r, lse_c = run.ws("lse_r", torch.float32, B, npad), run.ws("lse_c", torch.float32, B, npad)
    inv_t = 1.0 / run.cfg["FEATURE_MATCHER"]["DUAL_SOFTMAX"]["TEMPERATURE"]
    k2 = inv_t / math.log(2)
    dust = float(run.w("dustbin")) / math.log(2)
    d = run.data
    scr = torch.cat([d["scr0"], d["scr1"]], 0)[:, 0].double()
    # the 32-column chunk of the next row: row 500, columns 512..543 where the matrix holds them; on small grids the
    # first interior row (its final_scores row is zero outside the interior columns, which the chunk covers)
    sw_r, sw_c = (500, 512) if N > 600 else (run.interior, max(0, min(run.interior, N - 32)))
    # engine.cu run_match: fixed-shift partials for unit-norm descriptors while 1 / T <= 25, true maxima otherwise; the
    # bounds below hold in both modes
    mode = "fixed-shift partials" if run.norm_dsc and inv_t <= 25.0 else "online-max partials"
    tag = f"{run.name} ({mode}, {'with' if run.use_dustbin else 'without'} dustbin)"
    w_l = w_s = w_f = 0.0
    dust_planted = 0

    def lse2(v, dim):
        return torch.logsumexp(v * math.log(2), dim) / math.log(2)

    for p in range(B):
        a, b = DSCX[p].double(), DSCX[B + p].double()
        d0, d1 = a[:, :128] + a[:, 128:256], b[:, :128] + b[:, 256:]
        S = d0 @ d1.t()
        dS = 384 * 2.0 ** -23 * (a.abs() @ b.abs().t()) + a[:, 128:256].abs() @ b[:, 256:].abs().t()
        x = S * k2
        dx = k2 * dS + 2 * U32 * x.abs()
        xd = torch.full((1, 1), dust, dtype=torch.float64, device=DEV)
        lr_d, lc_d = lse2(torch.cat([x, xd.expand(N, 1)], 1), 1), lse2(torch.cat([x, xd.expand(1, N)], 0), 0)
        lr, lc = (lr_d, lc_d) if run.use_dustbin else (lse2(x, 1), lse2(x, 0))
        dlr = dx.amax(1) + ((N + 1) * U32 + 2.0 ** -22) / math.log(2) + 2.0 ** -22 * lr.abs()
        dlc = dx.amax(0) + ((N + 1) * U32 + 2.0 ** -22) / math.log(2) + 2.0 ** -22 * lc.abs()
        # the row (column) 40 unless the next one's lse is within its bound (flat logits at T = 1): then the one most apart
        rr, cc = _resolvable(lr, dlr), _resolvable(lc, dlc)
        muts = [ew.Mutation("lse of the next row", (slice(rr, rr + 1),), lr[rr + 1:rr + 2])]
        if not run.use_dustbin:
            # the dustbin column included although USE_DUSTBIN is off, at the row where its share is largest; planted
            # where that share is above four times the row's bound
            i = int((lr_d - lr - 4 * dlr).argmax())
            if float(lr_d[i] - lr[i]) > 4 * float(dlr[i]):
                muts.append(ew.Mutation("dustbin included although USE_DUSTBIN is off", (slice(i, i + 1),), lr_d[i:i + 1]))
                dust_planted += 1
        w_l = max(w_l, check(run, "matcher_lse", f"{tag} lse_r pair {p}", lse_r[p, :N], lr, dlr, mutations=muts))
        w_l = max(w_l, check(run, "matcher_lse", f"{tag} lse_c pair {p}", lse_c[p, :N], lc, dlc,
                             mutations=[ew.Mutation("lse of the next column", (slice(cc, cc + 1),), lc[cc + 1:cc + 2])]))
        sc_ref = torch.exp2(2 * x - lr[:, None] - lc[None, :])
        rel = math.log(2) * (2 * dx + dlr[:, None] + dlc[None, :]) + 2.0 ** -22 + 4 * U32
        b_sc = sc_ref * rel + 2.0 ** -126
        mut = [ew.row_chunk_swap(sc_ref, *_swap_at(sc_ref, b_sc, sw_r, sw_c))]
        w_s = max(w_s, check(run, "matcher_scores", f"{tag} scores pair {p}", d["scores"][p], sc_ref, b_sc, mutations=mut))
        f_ref = sc_ref * scr[p][:, None] * scr[B + p][None, :]
        b_f = f_ref * (rel + 3 * U32) + 2.0 ** -126
        w_f = max(w_f, check(run, "matcher_final_scores", f"{tag} final_scores pair {p}", d["_final_scores_fused"][p],
                             f_ref, b_f, mutations=[ew.row_chunk_swap(f_ref, *_swap_at(f_ref, b_f, sw_r, sw_c))]))
        del S, dS, x, dx, sc_ref, f_ref
    # at T = 1 unit-norm descriptors bound every logit by 1, so the dustbin keeps a resolvable share of some row of each
    # pair (DESIGN §6e); colder temperatures and raw descriptors can push it below every bound
    assert run.use_dustbin or not (run.norm_dsc and run.temperature == 1.0) or dust_planted == B, \
        f"{tag}: the dustbin's share is not resolvable"
    if not run.use_dustbin:
        print(f"\n[{run.name}] dustbin-included mutation planted in {dust_planted}/{B} pairs", end="")
    rec(run, "matcher_lse", w_l)
    rec(run, "matcher_scores", w_s)
    rec(run, "matcher_final_scores", w_f)
    # the pitched outputs' pad columns stay untouched: rerun the matcher (it reads only DSCX and the score copies) into
    # sentinel-filled buffers
    pitch = nn_pitch(N)
    outs = [torch.full((B, N, pitch), -7.0, device=DEV) for _ in range(3)]
    eng = run.eng
    _lib.check(eng.lib.mk_match(eng.h, B, _lib.ptr(outs[0]), _lib.ptr(outs[1]), _lib.ptr(outs[2]), pitch, _lib.ptr(eng.ws),
                                eng.ws.numel(), stream()), "mk_match")
    torch.cuda.synchronize()
    n4 = (N + 3) // 4 * 4
    for o, ref in zip(outs, (d["scores"], d["kp_scores"], d["_final_scores_fused"])):
        assert torch.equal(o[:, :, :N], ref)
        assert bool((o[:, :, n4:] == -7.0).all()), "pad columns were written"
        assert bool(((o[:, :, N:n4] == -7.0) | (o[:, :, N:n4] == 0.0)).all())


# ---------------------------------------------------------------------------------------------------------------
# §4: GEMMs whose inputs the workspace overwrites later in the call, relaunched on the workspace's operands
# ---------------------------------------------------------------------------------------------------------------
def _assert_regime(run, tiles: ew.GemmTiles, stage):
    if run.regime == "persistent":
        assert tiles.persistent, f"{stage}: {tiles.tiles} tiles no longer reach the persistent kernel at {run.name}"
    if run.regime == "one tile":
        assert not tiles.persistent, f"{stage}: {tiles.tiles} tiles no longer run one tile per CTA at {run.name}"


def relaunch_patch_embed(run):
    D, Mp, N, T = run.D, run.Mp, run.N, run.T
    P = run.ws("P", torch.float16, Mp, 640)
    Wp, posb = run.w("patch.w"), run.w("patch.posb")
    tiles = run.tiles(Mp, D)
    _assert_regime(run, tiles, "patch_embed")
    X = torch.full((run.M + 8, D + 32), 7.0, device=DEV)
    gemm("PATCH", P, Wp, Mp, D, 640, aux=posb, tok_per_img=N, out_f=X, out_f_ld=D + 32)
    torch.cuda.synchronize()
    Xv = X[:run.M].reshape(run.n_img, T, D + 32)
    assert bool((Xv[:, 0] == 7.0).all()) and bool((X[run.M:] == 7.0).all()) and bool((X[:, D:] == 7.0).all())
    Wd = Wp.double()
    worst = 0.0
    for i0, i1 in _chunks(run.n_img, 8):
        a = P[i0 * N:i1 * N].double()
        pre = a @ Wd.t()
        ref = pre + posb.double().repeat(i1 - i0, 1)
        bound = ew.gemm_acc_bound(640, a.abs() @ Wd.abs().t()) + ew.epilogue_terms(pre, posb.double().repeat(i1 - i0, 1)) + ew.out_rounding(ref, False)
        got = Xv[i0:i1, 1:, :D].reshape(-1, D)
        muts = [ew.Mutation("token of the neighbouring image", (slice(3, 4),), ref[N + 3:N + 4]),
                ew.Mutation("position embedding of the next token", (slice(3, 4),), (pre[3:4] + posb[4:5].double()))] if i1 - i0 > 1 else []
        worst = max(worst, check(run, "relaunch.patch_embed", f"{run.name} patch_embed", got, ref, bound.clamp_min(1e-30),
                                 ew.matrix_where(run.rows("patches"), tiles, row_offset=i0 * N), muts))
    rec(run, "relaunch.patch_embed", worst)


def relaunch_vit_linears(run):
    D, M = run.D, run.M
    blk = f"blk{run.depth - 1}."
    XN, ATT, H1 = run.ws("XN", torch.float16, M, D), run.ws("ATT", torch.float16, M, D), run.ws("H1", torch.float16, M, 4 * D)
    X = run.ws("X", torch.float32, M, D)
    # attn.qkv (EPI_STORE_H), sentinel rows and columns past the end
    tiles = run.tiles(M, 3 * D)
    _assert_regime(run, tiles, "attn.qkv")
    out = torch.full((M + 8, 3 * D + 64), 7.0, dtype=torch.float16, device=DEV)
    gemm("STORE_H", XN, run.w(blk + "qkv.w"), M, 3 * D, D, bias=run.w(blk + "qkv.b"), out_h=out, out_h_ld=3 * D + 64)
    torch.cuda.synchronize()
    assert bool((out[M:] == 7.0).all()) and bool((out[:, 3 * D:] == 7.0).all())
    _linear_check(run, "relaunch.attn_qkv", XN, run.w(blk + "qkv.w"), run.w(blk + "qkv.b"), out[:M, :3 * D], tiles=tiles)
    # attn.proj and mlp.fc2 (EPI_RESID_F, LayerScale) into copies of X
    for stage, A, wn, bn, gn, K in (("relaunch.attn_proj", ATT, "proj.w", "proj.b", "ls1", D),
                                    ("relaunch.mlp_fc2", H1, "fc2.w", "fc2.b", "ls2", 4 * D)):
        tiles = run.tiles(M, D)
        _assert_regime(run, tiles, stage)
        Xc = torch.full((M + 8, D + 32), 7.0, device=DEV)
        Xc[:M, :D] = X
        x0 = Xc[:M, :D].clone()
        gemm("RESID_F", A, run.w(blk + wn), M, D, K, bias=run.w(blk + bn), gamma=run.w(blk + gn), out_f=Xc, out_f_ld=D + 32)
        torch.cuda.synchronize()
        assert bool((Xc[M:] == 7.0).all()) and bool((Xc[:, D:] == 7.0).all())
        _linear_check(run, stage, A, run.w(blk + wn), run.w(blk + bn), Xc[:M, :D], fp16_out=False, tiles=tiles,
                      resid=x0, gamma=run.w(blk + gn))


def relaunch_head_gemms(run):
    R = run.R
    CAT, HM = run.ws("CAT", torch.float16, R, G * 256), run.ws("HM", torch.float16, R, G * 256)
    X32 = run.ws("X32", torch.float32, R, G * 128)
    # att.qkv: EPI_STORE_F, 4 groups reading their own 128 columns of CAT
    tiles = run.tiles(R, 384, G)
    _assert_regime(run, tiles, "att.qkv")
    out = torch.full((R + 8, G * 384), 7.0, device=DEV)
    Wq = run.w("att2.qkv.w")
    gemm("STORE_F", CAT, Wq, R, 384, 128, groups=G, a_col_group_off=256, b_row_group_off=384, out_f=out, out_f_ld=G * 384,
         out_f_group_off=384)
    # att.mlp0: EPI_STORE_H + ReLU over all 256 columns of each group
    tiles0 = run.tiles(R, 256, G)
    _assert_regime(run, tiles0, "att.mlp0")
    out0 = torch.full((R + 8, G * 256), 7.0, dtype=torch.float16, device=DEV)
    W0 = run.w("att2.mlp0.w")
    gemm("STORE_H", CAT, W0, R, 256, 256, groups=G, a_col_group_off=256, b_row_group_off=256, act=2, out_h=out0,
         out_h_ld=G * 256, out_h_group_off=256)
    torch.cuda.synchronize()
    assert bool((out[R:] == 7.0).all()) and bool((out0[R:] == 7.0).all())
    zero_b = lambda n: torch.zeros(n, device=DEV)                    # noqa: E731
    w1 = w2 = 0.0
    for g in range(G):
        w1 = max(w1, _linear_check(run, "relaunch.att_qkv", CAT[:, g * 256:g * 256 + 128], Wq[g * 384:(g + 1) * 384], zero_b(384),
                                   out[:R, g * 384:(g + 1) * 384], fp16_out=False, tiles=tiles, rows="padded", row_chunk=32768,
                                   group=g))
        w2 = max(w2, _linear_check(run, "relaunch.att_mlp0", CAT[:, g * 256:(g + 1) * 256], W0[g * 256:(g + 1) * 256], zero_b(256),
                                   out0[:R, g * 256:(g + 1) * 256], act="relu", tiles=tiles0, rows="padded", row_chunk=32768,
                                   group=g))
    rec(run, "relaunch.att_qkv", w1)
    rec(run, "relaunch.att_mlp0", w2)
    # att.mlp2_ln: EPI_LN with the residual (a copy of X32) and pad zeroing (always one tile per CTA: its epilogue
    # needs more registers than the persistent epilogue warps have)
    W2, n2w, n2b = run.w("att2.mlp2.w"), run.w("att2.n2.w"), run.w("att2.n2.b")
    xc = torch.full((R + 8, G * 128), 7.0, device=DEV)
    xc[:R] = X32
    x0 = X32.double()
    oh = torch.full((R + 8, G * 256), 7.0, dtype=torch.float16, device=DEV)
    gemm("LN", HM, W2, R, 128, 256, groups=G, a_col_group_off=256, b_row_group_off=128, gamma=n2w, beta=n2b, ln_group_off=128,
         eps=1e-5, out_f=xc, out_f_ld=G * 128, out_f_group_off=128, out_h=oh, out_h_ld=G * 256, out_h_group_off=256,
         pad_h2=run.h2, pad_w2=run.w2)
    torch.cuda.synchronize()
    assert bool((xc[R:] == 7.0).all()) and bool((oh[R:] == 7.0).all())
    assert bool((oh[:R].reshape(R, G, 256)[:, :, 128:] == 7.0).all()), "mlp2_ln wrote the merge half of CAT"
    worst = 0.0
    v = run.valid[:, None]
    for g in range(G):
        Wg = W2[g * 128:(g + 1) * 128].double()
        for r0, r1 in _chunks(R, 32768):
            a = HM[r0:r1, g * 256:(g + 1) * 256].double()
            acc = a @ Wg.t()
            y, b = ew.ln_bound(acc, ew.gemm_acc_bound(256, a.abs() @ Wg.abs().t()), n2w[g * 128:(g + 1) * 128].double(),
                               n2b[g * 128:(g + 1) * 128].double(), 1e-5)
            res = x0[r0:r1, g * 128:(g + 1) * 128]
            ref = torch.where(v[r0:r1], res + y, torch.zeros_like(y))
            bd = torch.where(v[r0:r1], b + ew.epilogue_terms(res, y, ref) + ew.out_rounding(ref, False), torch.zeros_like(b)).clamp_min(1e-30)
            muts = [ew.row_chunk_swap(ref, int(run.valid[r0:r1].nonzero()[5]), 32)] if g == G - 1 and r0 == 0 else []
            where = ew.Where(lambda idx, g=g: (int(idx[0]), g, int(idx[1])), run.rows("padded"), None, r0)
            worst = max(worst, check(run, "relaunch.mlp2_ln", f"{run.name} relaunch mlp2_ln X32", xc[r0:r1, g * 128:(g + 1) * 128],
                                     ref, bd, where, muts))
    assert torch.equal(oh[:R].reshape(R, G, 256)[:, :, :128], xc[:R].reshape(R, G, 128).half())
    rec(run, "relaunch.mlp2_ln", worst)


def relaunch_rb3_conv2(run):
    """rb3 conv2 with the S3 shortcut, PE on the groups of aux_group_mask, fp16 into a CAT-shaped buffer (the merge half
    of every group keeps its sentinel) and fp32 into an X32-shaped buffer."""
    R, co = run.R, run.bd[2]
    T3, S3 = run.ws("T3", torch.float16, R, G * co), run.ws("S3", torch.float16, R, G * co)
    pe = run.w("head.pe")
    c = run.eng.mkcfg
    mask = (0x7 if c.kp_pos_enc else 0) | (0x8 if c.dsc_pos_enc else 0)
    tiles = run.tiles(R, co, G)
    _assert_regime(run, tiles, "rb3.conv2")
    oh = torch.full((R + 8, G * 256), 7.0, dtype=torch.float16, device=DEV)
    of = torch.full((R + 8, G * 128), 7.0, device=DEV)
    taps = [(ky - 1) * run.w2 + (kx - 1) for ky in range(3) for kx in range(3)]
    gemm("CONV", T3, run.w("rb3.c2.w"), R, co, taps=taps, chunks_per_tap=co // 64, groups=G, a_col_group_off=co,
         b_row_group_off=co, bias=run.w("rb3.c2.b"), bias_group_off=co, res_h=S3, res_h_ld=G * co, res_h_group_off=co,
         act=2, pad_h2=run.h2, pad_w2=run.w2, out_h=oh, out_h_ld=G * 256, out_h_group_off=256, out_f=of, out_f_ld=G * 128,
         out_f_group_off=128, aux=pe, aux_group_mask=mask)
    torch.cuda.synchronize()
    assert bool((oh[R:] == 7.0).all()) and bool((of[R:] == 7.0).all())
    assert bool((oh[:R].reshape(R, G, 256)[:, :, 128:] == 7.0).all())
    pe_groups = [g for g in range(G) if (mask >> g) & 1]
    kw = dict(a_col0=lambda g: g * co, bias=run.w("rb3.c2.b"), res_of=lambda g, r0, r1: S3[r0:r1, g * co:(g + 1) * co],
              pe=pe, pe_groups=pe_groups)
    check_conv(run, "relaunch.rb3_conv2_f32", T3, co, run.w("rb3.c2.w"), G, co, True,
               lambda g, r0, r1: of[r0:r1, g * 128:(g + 1) * 128], fp16_out=False, **kw)
    check_conv(run, "relaunch.rb3_conv2_f16", T3, co, run.w("rb3.c2.w"), G, co, True,
               lambda g, r0, r1: oh[r0:r1, g * 256:g * 256 + 128], **kw)


# ---------------------------------------------------------------------------------------------------------------
# the solver's draws on a compute_matches result
# ---------------------------------------------------------------------------------------------------------------
class Solved:
    """The solver with its own draws on the final_scores of a compute_matches call, as forward() feeds it."""

    def __init__(self, name, cfg, model, data, B, im, ir):
        self.name, self.cfg, self.model, self.B, self.im, self.ir = name, cfg, model, B, im, ir
        self.data = dict(data)
        self.data["final_scores"] = self.data.pop("_final_scores_fused")
        with torch.no_grad():
            self.R, self.t, self.inl = model.e2e_Procrustes.estimate_pose_vectorized(self.data, seed=SEED)
        torch.cuda.synchronize()
        self.res = self.data["_solver"]
        self.hyp_Rt = model._engine().ws_view("hyp_Rt", torch.float32, (B * im * ir, 12)).clone()
        self.fs = self.data["final_scores"]
        self.N = self.fs.shape[-1]


def band_all(fs_b, got, b, IM, seed, label, n_s=N_S):
    """Band-check IM streams of n_s cells of pair b; returns (max n_diff, max n_band)."""
    p = fs_b.reshape(-1).double()
    worst_diff = worst_band = 0
    for s, key in draws.outer_keys(p, seed, b, range(IM)):
        r = draws.band_check(got[s], key, n_s)
        assert r["ok"], (label, b, s, r)
        worst_diff, worst_band = max(worst_diff, r["n_diff"]), max(worst_band, r["n_band"])
    return worst_diff, worst_band


def outer_draws_are_the_race(sol):
    """Every stream is the fp64 race's top 2048 up to the key band; a pair with fewer than 2048 positive cells draws
    every positive cell plus the lowest-index zero cells (DESIGN §2)."""
    assert int(sol.res["status"].item()) == 0
    got = sol.res["sampled_idx"].long().reshape(sol.B, sol.im, N_S)
    diff = band = filled = 0
    for b in range(sol.B):
        pb = sol.fs[b].contiguous().reshape(-1)
        if int((pb > 0).sum()) < N_S:
            want = draws.fill_draw(pb, N_S)
            assert all(torch.equal(got[b, s], want) for s in range(sol.im)), (sol.name, b)
            filled += sol.im
            continue
        d, n = band_all(sol.fs[b].contiguous(), got[b], b, sol.im, SEED, sol.name)
        diff, band = max(diff, d), max(band, n)
    print(f"\n[{sol.name}] {sol.B * sol.im} streams ({filled} by the fill rule): max cells differing from fp64 {diff}, "
          f"max cells in band {band}")


def inner_draws_are_restated(sol):
    """Every inner triple restated bit for bit; hyp_Rt and hyp_scores against an fp64 Kabsch and soft count of it; the
    pose against the fp64 oracle's with both of the kernel's draws injected."""
    B, im, ir = sol.B, sol.im, sol.ir
    outer = sol.res["sampled_idx"].long()                               # [B*im, n_s]
    b_of = torch.arange(B, device=DEV).repeat_interleave(im)
    s_in = torch.arange(im, device=DEV).repeat(B)
    w = sol.fs.reshape(B, -1)[b_of[:, None], outer]
    idx, amb = draws.inner_draw(draws.inner_cdf(w.float()), SEED, b_of, s_in, ir)
    inner = idx.reshape(-1, 3)
    d = sol.data
    tr = {}
    Ro, to, _ = mo.solve_pose(sol.fs.double(), d["kps0"].double(), d["depth_kp0"].double(), d["kps1"].double(),
                              d["depth_kp1"].double(), d["K_color0"].double(), d["K_color1"].double(), sol.cfg,
                              outer_idx=outer, inner_idx=inner, trace=tr)
    X, Y = tr["X"], tr["Y"]
    s_of = torch.arange(B * im, device=DEV).repeat_interleave(ir)

    def kabsch_of(inn):
        Xk, Yk = X[s_of[:, None], inn], Y[s_of[:, None], inn]
        Rr, tr_ = mo.kabsch(Xk, Yk)
        Hm = (Xk - Xk.mean(1, keepdim=True)).transpose(1, 2) @ (Yk - Yk.mean(1, keepdim=True))
        sv = torch.linalg.svdvals(Hm)
        return Rr.reshape(-1, 9), tr_.reshape(-1, 3), sv[:, 1] > 1e-3 * sv[:, 0]

    Rr, tr_, well = kabsch_of(inner)
    well &= ~amb.reshape(-1)
    assert float(well.float().mean()) > 0.5
    got = sol.hyp_Rt.double()
    bound_R, bound_t = 1e-3, 1e-3 * (1 + tr_.abs())

    def misses(R_, t_):
        return ((got[:, :9] - R_).abs().amax(1) > bound_R) | ((got[:, 9:] - t_).abs() > bound_t).any(1)

    miss = misses(Rr, tr_) & well
    assert int(miss.sum()) == 0, (sol.name, int(miss.sum()), int(well.sum()))
    # power: one triple member replaced by its neighbour in the set
    mut = inner.clone()
    mut[:, 0] = (mut[:, 0] + 1) % N_S
    Rm, tm, well_m = kabsch_of(mut)
    rej = misses(Rm, tm)[well & well_m]
    assert float(rej.float().mean()) > 0.9, float(rej.float().mean())
    # soft inlier counts (the bound of test_solver_production_batch_injected_draws)
    hyp, ref = sol.res["hyp_scores"].double(), tr["hyp_scores"].double()
    wl = well.reshape(hyp.shape)
    assert bool(((hyp - ref).abs() <= 1e-3 * ref.abs() + 1e-3)[wl].all())
    # the pose: a tie-tolerant winner, and the oracle's pose where the winner is the same
    win = hyp.argmax(1)
    assert bool((ref.gather(1, win[:, None])[:, 0] >= ref.max(1).values * (1 - 1e-3)).all())
    same = win == tr["best"]
    if bool(same.any()):
        assert float(rotation_angle_deg(sol.R[same].double(), Ro.reshape(B, 3, 3)[same]).max()) < 1e-2
        assert float((sol.t.reshape(B, 3)[same].double() - to.reshape(B, 3)[same]).abs().max()) < 1e-3
    print(f"\n[{sol.name}] {inner.shape[0]} hypotheses: {int(amb.sum())} ambiguous, {int(well.sum())} checked, "
          f"neighbour mutation rejected in {float(rej.float().mean()):.4f}, same winner in {int(same.sum())}/{B} pairs")
