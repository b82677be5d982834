"""Every kernel stage at production geometry, element by element against fp64, on the engine's own intermediates.

Three module-scoped runs of `compute_matches` on 720x540 synthetic pairs:
  C2: ViT-S, 1 pair (one-tile and deep-ring GEMM launches)     C3: ViT-B, 32 pairs (persistent GEMMs, multi-wave attention,
  L:  ViT-L, 1 pair (D = 1024, 16 heads, K = 4096 fc2)             the 32-pair matcher)
The checks themselves are in tests/stages.py (the same harness runs at other image sizes in
tests/test_gpu_stages_geometries.py).  `max(err / bound)` per stage goes to $MICKEY_STAGE_METRICS (a JSON file) when set.
"""
import pytest
import torch

from mickey_b200.config import mickey_cfg
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from oracle import mickey_oracle as mo
from tests import elementwise as ew
from tests import stages as st
from tests.common import rotation_angle_deg
from tests.planted import planted_problem

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, W = 720, 540
GEOS = {"C2": ("vits", 1, 8, 64, "one tile"), "C3": ("vitb", 32, 16, 64, "persistent"), "L": ("vitl", 1, 20, 100, None)}


@pytest.fixture(scope="module", params=list(GEOS))
def run(request):
    variant, B, im, ir, regime = GEOS[request.param]
    r = st.Run(request.param, variant, B, H, W, im, ir, regime)
    yield r
    del r
    torch.cuda.empty_cache()


def test_patch_gather(run):
    st.patch_gather(run)


def test_final_layernorm_and_scatter(run):
    st.final_layernorm_and_scatter(run)


def test_last_block_attention(run):
    st.last_block_attention(run)


def test_last_block_fc1_gelu(run):
    st.last_block_fc1_gelu(run)


def test_head_residual_blocks(run):
    st.head_residual_blocks(run)


def test_linear_attention_last_layer(run):
    st.linear_attention_last_layer(run)


def test_head_transformer_outputs(run):
    st.head_transformer_outputs(run)


def test_block4(run):
    st.block4(run)


def test_head_outputs(run):
    st.head_outputs(run)


def test_matcher(run):
    st.matcher(run)


def test_relaunch_patch_embed(run):
    st.relaunch_patch_embed(run)


def test_relaunch_vit_linears(run):
    st.relaunch_vit_linears(run)


def test_relaunch_head_gemms(run):
    st.relaunch_head_gemms(run)


def test_relaunch_rb3_conv2(run):
    st.relaunch_rb3_conv2(run)


# ---------------------------------------------------------------------------------------------------------------
# §5: the solver at production batch, planted problems with host-drawn indices, against the fp64 oracle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,im,ir", [(32, 16, 64), (3, 20, 100)])
def test_solver_production_batch_injected_draws(B, im, ir):
    cfg = mickey_cfg("vits", im, ir)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    model = model.cuda().eval()
    gh, gw = 51, 38
    N = gh * gw
    eng = model._engine()
    eng._ws_for(B, 14 * gh, 14 * gw)
    prob = planted_problem(n_side=(gh, gw), batch=B, outlier_frac=0.4, seed=2)
    n_s = cfg.PROCRUSTES.NUM_SAMPLED_MATCHES
    g = torch.Generator().manual_seed(11)
    outer = []
    for s in range(B * im):
        diag = torch.randperm(N, generator=g)[:n_s - 64]
        cells = torch.cat([diag * (N + 1), torch.randint(0, N * N, (64,), generator=g)])
        cells = torch.unique(cells)
        while cells.numel() < n_s:
            cells = torch.unique(torch.cat([cells, torch.randint(0, N * N, (n_s - cells.numel(),), generator=g)]))
        outer.append(cells[:n_s])
    outer = torch.stack(outer).long()
    inner = torch.rand(B * im * ir, n_s, generator=g).topk(3, dim=1).indices.long()
    trace = {}
    Ro, to, _ = mo.solve_pose(prob["final_scores"].double(), prob["kps0"].double(), prob["depth0"].double(),
                              prob["kps1"].double(), prob["depth1"].double(), prob["K"].double(), prob["K"].double(), cfg,
                              outer_idx=outer, inner_idx=inner, trace=trace)
    batch = {"final_scores": prob["final_scores"].to(DEV), "kps0": prob["kps0"].to(DEV), "kps1": prob["kps1"].to(DEV),
             "depth_kp0": prob["depth0"].to(DEV), "depth_kp1": prob["depth1"].to(DEV), "K_color0": prob["K"].to(DEV),
             "K_color1": prob["K"].to(DEV)}
    R, t, _ = model.e2e_Procrustes.estimate_pose_vectorized(batch, outer_idx=outer.int(), inner_idx=inner.int())
    res = batch["_solver"]
    torch.cuda.synchronize()
    assert int(res["status"].item()) == 0
    hyp, ref = res["hyp_scores"].double().cpu(), trace["hyp_scores"].double()
    # well-conditioned 3-point samples only (a rank-1 centred covariance has no unique Kabsch optimum)
    X, Y, inn = trace["X"], trace["Y"], trace["inner_idx"]
    s_of = torch.arange(X.shape[0]).repeat_interleave(ir)
    Xk, Yk = X[s_of[:, None], inn].double(), Y[s_of[:, None], inn].double()
    Hm = (Xk - Xk.mean(1, keepdim=True)).transpose(1, 2) @ (Yk - Yk.mean(1, keepdim=True))
    sv = torch.linalg.svdvals(Hm)
    well = (sv[:, 1] > 1e-3 * sv[:, 0]).reshape(hyp.shape)
    assert float(well.float().mean()) > 0.5
    # a soft inlier count of an fp32 three-point pose: relative 1e-3 (plus 1e-3 of one inlier)
    r = ew.check(f"solver B={B} hyp_scores", hyp[well], ref[well], 1e-3 * ref[well].abs() + 1e-3)
    ew.record(f"solver_hyp_scores_B{B}_{im}x{ir}", "solver", r)
    win = hyp.argmax(1)
    tied = ref.gather(1, win[:, None])[:, 0] >= ref.max(1).values * (1 - 1e-3)
    assert bool(tied.all())
    assert float(rotation_angle_deg(R, prob["R"]).max()) < 0.1 and float((t.cpu() - prob["t"]).abs().max()) < 5e-3
    same = win == trace["best"]                                     # pairs whose winner is the oracle's
    R, t = R.cpu()[same], t.cpu().reshape(B, 3)[same].double()
    if bool(same.any()):
        assert float(rotation_angle_deg(R, Ro.reshape(B, 3, 3)[same]).max()) < 1e-2
        assert float((t - to.reshape(B, 3)[same].double()).abs().max()) < 1e-3
