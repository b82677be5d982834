"""The handle-free pose solver (mk_procrustes_solve, mickey_b200/procrustes.py) on the GPU.

1. Same kernels, same bits: against MickeyRelativePose's engine-bound solver (mk_solve_pose) on the same tensors with
   the same seed, on the engine's pitch-1952 view and on a contiguous copy.
2. The training model's validation shapes (B = 8, N = 1938 and B = 24, N = 850, final_scores a contiguous scores *
   kp_scores at pitch N) against the fp64 oracle: with the oracle's draws injected, and with the kernel's own draws
   (every outer stream the race up to the key band, every inner triple restated bit for bit).
3. The zero result exactly where the oracle (and torch.multinomial) gives it.
4. A converted MicKeyTrainingModel's validation_step and its logging call with the solver swapped in.
5. The call's peak allocation at B = 24, N = 850.
"""
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.loss import vcre_grid
from mickey_b200.model import MickeyRelativePose
from mickey_b200.procrustes import e2eProbabilisticProcrustesSolver
from mickey_b200.training import use_cuda_modules
from mickey_b200.weights import synthetic_state_dict
from oracle import mickey_oracle as mo
from tests import draws, planted, stages
from tests.common import rotation_angle_deg, synthetic_pair
from tests.test_gpu_heads_training import STEP_CASES, converted_model, step_batch
from tests.test_gpu_training_lifecycle import validation_step

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = stages.SEED
N_S = 2048
KEYS = ("pose", "best_set", "inlier_mask", "sampled_idx", "hyp_scores", "status")


def solve(solver, batch, **kw):
    """estimate_pose_vectorized with return_inliers and the solver's outputs."""
    b = dict(batch)
    R, t, inl, lst = solver.estimate_pose_vectorized(b, return_inliers=True, **kw)
    torch.cuda.synchronize()
    return R, t, inl, lst, b["_solver"]


def assert_same(a, b):
    Ra, ta, ia, la, sa = a
    Rb, tb, ib, lb, sb = b
    assert torch.equal(Ra, Rb) and torch.equal(ta, tb) and torch.equal(ia, ib)
    assert all(torch.equal(sa[k], sb[k]) for k in KEYS), [k for k in KEYS if not torch.equal(sa[k], sb[k])]
    assert len(la) == len(lb) and all(torch.equal(x, y) for x, y in zip(la, lb))


# ---- 1. the engine-bound solver's bits ---------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [2, 32])
def test_same_bits_as_the_engine_bound_solver(B):
    cfg = mickey_cfg("vits", 20, 100)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
    model = model.cuda().eval()
    data = {k: v.to(DEV) for k, v in synthetic_pair(B, 720, 540, seed=17).items()}
    with torch.no_grad():
        model.compute_matches(data)
    data["final_scores"] = data.pop("_final_scores_fused")
    assert data["final_scores"].stride(1) == 1952
    ours = e2eProbabilisticProcrustesSolver(cfg)
    for s in (SEED, 12345):
        ref = solve(model.e2e_Procrustes, data, seed=s)
        assert int(ref[4]["status"].item()) == 0
        assert_same(ours_out := solve(ours, data, seed=s), ref)
        assert ours_out[2].shape == (B, 1) and all(x.shape[1] == 7 for x in ours_out[3])
        assert_same(solve(ours, dict(data, final_scores=data["final_scores"].contiguous()), seed=s), ref)


# ---- 2. the validation shapes against fp64 ----------------------------------------------------------------------------
TRAINING_SHAPES = {"b8_720x540": (8, 51, 38), "b24_480x360": (24, 34, 25)}


def training_batch(B, gh, gw, seed=0):
    """A planted pose per pair (tests/planted.py) with keypoint i of image 0 matching keypoint i of image 1, and
    final_scores as the training model builds it (model.py:198-203): the dual softmax of descriptors that match along
    the diagonal, times the outer product of the keypoint scores, contiguous at pitch N."""
    p = planted.planted_problem((gh, gw), batch=B, seed=seed)
    N = gh * gw
    g = torch.Generator(device=DEV).manual_seed(seed)
    d0 = torch.nn.functional.normalize(torch.randn(B, 128, N, generator=g, device=DEV), dim=1)
    d1 = torch.nn.functional.normalize(d0 + 0.05 * torch.randn(B, 128, N, generator=g, device=DEV), dim=1)
    scr0 = torch.rand(B, 1, N, generator=g, device=DEV)
    scr1 = torch.rand(B, 1, N, generator=g, device=DEV)
    scores = mo.dual_softmax(d0, d1, 0.1, torch.tensor(1.0, device=DEV))
    final = scores * torch.matmul(scr0.transpose(2, 1), scr1)
    assert final.is_contiguous()
    K = p["K"].to(DEV)
    return {"final_scores": final, "kps0": p["kps0"].to(DEV), "kps1": p["kps1"].to(DEV),
            "depth_kp0": p["depth0"].to(DEV), "depth_kp1": p["depth1"].to(DEV), "K_color0": K, "K_color1": K}


def oracle(batch, cfg, **kw):
    d = batch
    tr = {}
    R, t, inl = mo.solve_pose(d["final_scores"].double(), d["kps0"].double(), d["depth_kp0"].double(), d["kps1"].double(),
                              d["depth_kp1"].double(), d["K_color0"].double(), d["K_color1"].double(), cfg, trace=tr, **kw)
    return R, t, inl, tr


def check_against_oracle(ours, ref, B, label):
    """Hypothesis scores, and the pose and inliers where the winner is the same (DESIGN §2 bounds)."""
    R, t, inl, _, res = ours
    Ro, to, inlo, tr = ref
    hyp, refh = res["hyp_scores"].double(), tr["hyp_scores"].double()
    assert bool(((hyp - refh).abs() <= 1e-3 * refh.abs() + 1e-3).all()), label
    win = hyp.argmax(1)
    assert bool((refh.gather(1, win[:, None])[:, 0] >= refh.max(1).values * (1 - 1e-3)).all()), label
    same = win == tr["best"]
    assert float(rotation_angle_deg(R[same].double(), Ro.reshape(B, 3, 3)[same]).max()) < 1e-2, label
    assert float((t.reshape(B, 3)[same].double() - to.reshape(B, 3)[same]).abs().max()) < 1e-3, label
    io = inlo.reshape(B)[same]
    assert bool(((inl.reshape(B)[same].double() - io).abs() <= 1e-3 * io.abs() + 1e-3).all()), label
    return int(same.sum())


@pytest.fixture(scope="module", params=list(TRAINING_SHAPES))
def shape(request):
    B, gh, gw = TRAINING_SHAPES[request.param]
    yield request.param, B, gh * gw, training_batch(B, gh, gw)
    torch.cuda.empty_cache()


def test_validation_shapes_with_the_oracles_draws(shape):
    name, B, N, batch = shape
    cfg = mickey_cfg("vitl")
    g = torch.Generator(device=DEV).manual_seed(B)
    ref = oracle(batch, cfg, generator=g)
    tr = ref[3]
    ours = solve(e2eProbabilisticProcrustesSolver(cfg), batch, outer_idx=tr["outer_idx"], inner_idx=tr["inner_idx"],
                 seed=SEED)
    assert int(ours[4]["status"].item()) == 0
    same = check_against_oracle(ours, ref, B, name)
    print(f"\n[{name}] oracle draws: same winner in {same}/{B} pairs")


def test_validation_shapes_with_the_kernels_draws(shape):
    name, B, N, batch = shape
    fs = batch["final_scores"]
    # neither pitch is 16-byte aligned, but every matrix is (N * N % 4 == 0): the flat vector loads
    assert N % 4 != 0 and fs.data_ptr() % 16 == 0
    assert stages.sampler_mode(N, N) == "FLAT_VEC"
    cfg = mickey_cfg("vitl")
    IM, IR = 20, 100
    solver = e2eProbabilisticProcrustesSolver(cfg)
    own = solve(solver, batch, seed=SEED)
    res = own[4]
    assert int(res["status"].item()) == 0
    outer = res["sampled_idx"].long()
    got = outer.reshape(B, IM, N_S)
    for b in range(B):
        stages.band_all(fs[b], got[b], b, IM, SEED, name)
    b_of = torch.arange(B, device=DEV).repeat_interleave(IM)
    w = fs.reshape(B, -1)[b_of[:, None], outer]
    idx, amb = draws.inner_draw(draws.inner_cdf(w.float()), SEED, b_of, torch.arange(IM, device=DEV).repeat(B), IR)
    inner = idx.reshape(-1, 3)
    # the restated triples, injected, give every unambiguous hypothesis's score bit for bit
    again = solve(solver, batch, outer_idx=outer, inner_idx=inner, seed=SEED)
    clear = ~amb.reshape(B, IM * IR)
    assert float(clear.float().mean()) > 0.99
    assert torch.equal(again[4]["hyp_scores"][clear], res["hyp_scores"][clear])
    if bool(clear.all()):
        assert_same(again, own)
    same = check_against_oracle(own, oracle(batch, cfg, outer_idx=outer, inner_idx=inner), B, name)
    print(f"\n[{name}] kernel draws: {int((~clear).sum())} ambiguous triples, same winner in {same}/{B} pairs")


# ---- 3. the zero result ------------------------------------------------------------------------------------------------
# case -> whether the reference gives the zero result.  The oracle and torch.multinomial run on the CPU, where torch
# raises on a bad distribution instead of asserting on the device.
ZERO_CASES = {"nan": True, "inf": True, "-inf": True, "negative": True, "pos0": True, "nan_depth": True,
              "pos1": False, "neg_zero": False}


def zero_case_matrix(case):
    if case in ("-inf", "nan_depth"):
        fs = draws.contract_matrix("neg_zero")
        if case == "-inf":
            fs[draws.CONTRACT_PAIR, 3, 5] = -float("inf")
        return fs
    return draws.contract_matrix(case)


@pytest.mark.parametrize("case", list(ZERO_CASES))
def test_zero_result_where_the_oracle_gives_it(case):
    cfg = mickey_cfg("vits", 2, 8)
    B, N, P = draws.CONTRACT_B, draws.CONTRACT_N, draws.CONTRACT_PAIR
    IM, IR = 2, 8
    fs = zero_case_matrix(case)
    kps0, d0, kps1, d1, K = draws.contract_geometry()
    kw = {}
    if case == "nan_depth":            # a NaN depth at a keypoint the injected draws use: a non-finite hypothesis (bit 2)
        g = torch.Generator().manual_seed(1)
        tiled = fs.reshape(B, 1, N * N).expand(B, IM, N * N).reshape(B * IM, N * N).clamp_min(0)
        outer = torch.multinomial(tiled, N_S, generator=g)
        inner = torch.rand(B * IM * IR, N_S, generator=g).argsort(1)[:, :3]
        d0 = d0.clone()
        d0[P, 0, int(outer[P * IM, int(inner[P * IM * IR, 0])]) // N] = float("nan")
        kw = dict(outer_idx=outer, inner_idx=inner)
    zero = ZERO_CASES[case]
    if zero:
        Ro, to, io, lo = mo.solve_pose(fs.double(), kps0.double(), d0.double(), kps1.double(), d1.double(), K.double(),
                                       K.double(), cfg, return_inliers=True, generator=torch.Generator().manual_seed(2),
                                       **kw)
        assert float(Ro.abs().max()) == 0 and float(to.abs().max()) == 0 and float(io.abs().max()) == 0
    if case != "nan_depth":            # the outer draw: torch refuses exactly the zero cases
        if zero:
            with pytest.raises(RuntimeError):
                torch.multinomial(fs.reshape(B, N * N), N_S)
        else:
            torch.multinomial(fs.reshape(B, N * N), N_S)
    batch = {k: v.to(DEV) for k, v in dict(final_scores=fs, kps0=kps0, kps1=kps1, depth_kp0=d0, depth_kp1=d1,
                                            K_color0=K, K_color1=K).items()}
    R, t, inl, lst, res = solve(e2eProbabilisticProcrustesSolver(cfg), batch, seed=SEED,
                                **{k: v.to(DEV) for k, v in kw.items()})
    status = int(res["status"].item())
    assert bool(status & 7) == zero, status
    if case == "nan_depth":
        assert status & 4
    if zero:
        assert torch.equal(R, torch.zeros(B, 3, 3, device=DEV)) and torch.equal(t, torch.zeros(B, 1, 3, device=DEV))
        assert torch.equal(inl, torch.zeros(B, device=DEV))
        assert len(lst) == B and all(x.shape == (0, 5) and x.device.type == "cpu" for x in lst)
    else:
        assert bool(torch.isfinite(R).all()) and float(R.abs().max()) > 0 and inl.shape == (B, 1)
        assert len(lst) == B and all(x.shape[1] == 7 for x in lst)


# ---- 4. the converted training model ------------------------------------------------------------------------------------
def pose_error(R, t, Tgt):
    """pose_error_torch (lib/utils/metrics.py:12-48) with reduce=None: translation angle (deg), euclidean error and
    rotation error (deg)."""
    Rgt, tgt = Tgt[:, :3, :3], Tgt[:, :3, 3:].transpose(1, 2)
    n, ngt = torch.linalg.norm(t, dim=-1), torch.linalg.norm(tgt, dim=-1)
    cos = torch.clip((t @ tgt.transpose(1, 2)).squeeze(-1) / (n * ngt + 1e-9), -1.0, 1.0)
    ang = torch.rad2deg(torch.acos(cos))
    ang = torch.minimum(ang, 180 - ang)
    tr = torch.diagonal(R.transpose(1, 2) @ Rgt, dim1=-2, dim2=-1).sum(-1)
    return {"t_err_ang": ang, "t_err_euc": torch.linalg.norm(t - tgt, dim=-1),
            "R_err": torch.rad2deg(torch.acos(torch.clip((tr - 1) / 2, -1.0, 1.0)))}


def vcre(R, t, Tgt, K0, H=720, W=540):
    """vcre_torch (lib/utils/metrics.py:83-124) with reduce=None: the mean reprojection error of the virtual grid."""
    B = R.shape[0]
    grid = vcre_grid(R.device).float()
    eye = torch.cat([grid, torch.ones_like(grid[:, :1])], 1)[None].expand(B, -1, -1)
    project = lambda X: (lambda xyz: (xyz / (xyz[:, :, 2:3] + 1e-16))[:, :, :2])((K0 @ X.transpose(2, 1)).transpose(2, 1))
    uv_gt = project(eye[:, :, :3])
    est = torch.eye(4, device=R.device).repeat(B, 1, 1)
    est[:, :3, :3], est[:, :3, 3] = R, t[:, 0]
    gt = torch.eye(4, device=R.device).repeat(B, 1, 1)
    gt[:, :3, :3], gt[:, :3, 3] = Tgt[:, :3, :3], Tgt[:, :3, 3]
    uv_pred = project((torch.linalg.inv(gt) @ est @ eye.transpose(2, 1)).transpose(2, 1)[:, :, :3])
    lim = torch.tensor([W, H], device=R.device, dtype=uv_gt.dtype)
    uv_gt, uv_pred = torch.minimum(uv_gt.clamp_min(0), lim), torch.minimum(uv_pred.clamp_min(0), lim)
    return ((((uv_gt - uv_pred) ** 2).sum(-1) + 1e-6) ** 0.5).mean(-1).view(B, 1)


def full_validation_step(model, ims, data, seed):
    """validation_step (model.py:66-89): the forward and the loss as test_gpu_training_lifecycle restates them, then the
    pose metrics from model.e2e_Procrustes."""
    _, _, batch, outputs, _ = validation_step(model, ims, data, seed)
    R, t, inl = model.e2e_Procrustes.estimate_pose_vectorized(batch, seed=seed + 1)
    m = pose_error(R, t, batch["T_0to1"])
    outputs.update(metric_ours_t_err_ang=m["t_err_ang"], metric_ours_t_err_euc=m["t_err_euc"],
                   metric_ours_R_err=m["R_err"], metric_inliers=inl,
                   metric_ours_vcre=vcre(R, t, batch["T_0to1"], batch["Kori_color0"]))
    return batch, outputs


def test_converted_model_validation_and_logging():
    config, B, H, W = STEP_CASES["vitl_224x210_b2_overlap_warm_up"]
    torch.manual_seed(0)
    model = use_cuda_modules(converted_model(config), solver=True)
    assert type(model.e2e_Procrustes) is e2eProbabilisticProcrustesSolver
    before = {k: v.clone() for k, v in model.state_dict().items()}
    assert all(p.grad is None for p in model.parameters())
    steps = []
    for i in range(2):
        ims, data = step_batch(B, H, W, seed=40 + i)
        with torch.inference_mode():
            batch, out_inf = full_validation_step(model, ims, data, seed=50 + i)
        _, out_grad = full_validation_step(model, ims, data, seed=50 + i)
        for k in [k for k in out_inf if k.startswith("metric")]:
            assert torch.equal(out_inf[k], out_grad[k].detach()), k
            assert not out_grad[k].requires_grad, k
        steps.append(out_inf)
        # the tensorboard_log_step call (model.py:164), in grad mode as in backward_step
        R, t, inl, lst = model.e2e_Procrustes.estimate_pose_vectorized(batch, return_inliers=True)
        assert len(lst) == B
        for x in lst:
            assert x.shape[0] == 0 or (x.shape[1] == 7 and x.device.type == "cuda" and bool(torch.isfinite(x).all()))
            assert bool((x[1:, 4] <= x[:-1, 4]).all()) and not x.requires_grad
    assert all(p.grad is None for p in model.parameters())
    after = model.state_dict()
    assert all(torch.equal(after[k], v) for k, v in before.items())
    # on_validation_epoch_end (model.py:205-234): stacked over the steps, every mean finite
    agg = {k: torch.stack([s[k] for s in steps]) for k in steps[0] if k.startswith("metric") or k in ("loss",)}
    assert all(bool(torch.isfinite(v.float().mean())) for v in agg.values()), {k: v.float().mean() for k, v in agg.items()}
    accepted = (agg["metric_ours_t_err_euc"].view(-1) < 0.25) * (agg["metric_ours_R_err"].view(-1) < 5)
    assert accepted.numel() == 2 * B and agg["metric_inliers"].view(-1).numel() == 2 * B


# ---- 5. memory -----------------------------------------------------------------------------------------------------------
def test_peak_allocation_at_b24_n850(shape):
    name, B, N, batch = shape
    if name != "b24_480x360":
        pytest.skip("one shape")
    cfg = mickey_cfg("vitl")
    IM, IR = 20, 100
    solver = e2eProbabilisticProcrustesSolver(cfg)
    solve(solver, batch, seed=SEED)                    # warm: the caching allocator's pools exist
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    R, t, inl, lst, res = solve(solver, batch, seed=SEED)
    peak = torch.cuda.max_memory_allocated() - base
    ws = _lib.load().mk_procrustes_ws_bytes(B, N, IM, IR, N_S)
    outputs = 4 * (B * 13 + B + B * N_S + B * IM * N_S + B * IM * IR + 1) + 4 * 2 * B * 3 * N + 4 * 2 * 9 * B
    lists = B * N_S * 128                                              # the inlier list's gathers and rows
    bound = ws + outputs + lists + (8 << 20)                           # 8 MB for the allocator's rounding
    tile = B * IM * N * N * 4
    print(f"\n[{name}] peak above inputs {peak / 2**20:.1f} MB, bound {bound / 2**20:.1f} MB, workspace "
          f"{ws / 2**20:.1f} MB, [B*IT_MATCHES, N^2] tile {tile / 2**30:.2f} GB")
    assert peak <= bound and peak < tile
