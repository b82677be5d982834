"""Every kernel stage, the solver's draws and the mutual matches at image geometries other than 720x540.

The production size gives every geometry-dependent quantity one value (N = 1938, T = 1939, a 51 x 38 portrait grid,
pitch 1952).  The runs here (tests/stages.py GEOMETRIES, synthetic weights, seed 3) reach the other sides of those
choices: a landscape grid with persistent GEMMs (land), npad = pitch = N and the sampler's flat loads (n1920), every
attention and GEMM M-tile full (t2304), crop margins filled with NaN (crop), the smallest image with one interior score
cell (min), the position embedding without interpolation (sq37) and N > 4096 (large).  Each stage check of
tests/test_gpu_stages_at_scale.py runs on each of them; `max(err / bound)` per stage goes to $MICKEY_STAGE_METRICS.
"""
import pytest
import torch

from mickey_b200.config import mickey_cfg
from mickey_b200.matches import MAX_N
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from oracle.matches_oracle import matches_list
from tests import draws
from tests import stages as st
from tests.common import synthetic_pair

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", params=list(st.GEOMETRIES))
def run(request):
    r = st.Run(request.param, *st.GEOMETRIES[request.param])
    yield r
    del r
    torch.cuda.empty_cache()


def test_geometry_paths(run):
    """The run reaches the paths GEOMETRY_PATHS names for it."""
    (gh, gw), N, pitch, mode = st.GEOMETRY_PATHS[run.name]
    fs = run.data["_final_scores_fused"]
    assert (run.gh, run.gw, run.N) == (gh, gw, N)
    assert fs.stride(1) == pitch and fs.stride(0) == N * pitch
    assert st.sampler_mode(N, fs.stride(1), fs.data_ptr() % 16 == 0) == mode


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


def test_solver_draws(run):
    """The engine's own outer draws and inner triples.  At `min` the matrix has one positive cell, so every stream is
    that cell plus the lowest-index zero cells, and every triple is that cell and the two entries after it (the
    guard's rule): its three kps0 points coincide, so the Kabsch problem is degenerate and there is no fp64 pose to
    compare with; every hypothesis of a stream must then give bit-identical hyp_Rt and scores."""
    sol = st.Solved(run.name, run.cfg, run.model, run.data, run.B, run.im, run.ir)
    st.outer_draws_are_the_race(sol)
    if run.name != "min":
        st.inner_draws_are_restated(sol)
        return
    pos = (sol.fs.reshape(-1) > 0).nonzero()[:, 0]
    assert pos.tolist() == [run.interior * run.N + run.interior]
    outer = sol.res["sampled_idx"].long()
    at = int((outer[0] == pos[0]).nonzero()[0])
    w = sol.fs.reshape(1, -1)[0, outer]
    idx, _ = draws.inner_draw(draws.inner_cdf(w), st.SEED, torch.zeros(run.im, dtype=torch.int64, device=DEV),
                              torch.arange(run.im, device=DEV), run.ir)
    assert bool((idx == torch.tensor([at, at + 1, at + 2], device=DEV)).all())
    Rt = sol.hyp_Rt.reshape(run.im, run.ir, 12)
    hyp = sol.res["hyp_scores"].reshape(run.im, run.ir)
    assert bool(torch.isfinite(Rt).all()) and bool((Rt == Rt[:, :1]).all()) and bool((hyp == hyp[:, :1]).all())
    assert bool(torch.isfinite(sol.R).all()) and bool(torch.isfinite(sol.t).all())


def test_mutual_matches(run):
    """model.mutual_matches on the run's final_scores equals the oracle exactly; beyond MAX_N it is rejected on the
    host."""
    fs = run.data["_final_scores_fused"]
    if run.N > MAX_N:
        with pytest.raises(ValueError, match="N <= 4097"):
            run.model.mutual_matches(fs)
        return
    lists, scores = run.model.mutual_matches(fs)
    for b in range(run.B):
        rm, rv = matches_list(fs[b].cpu())
        assert torch.equal(lists[b].cpu(), rm) and torch.equal(scores[b].cpu(), rv), (run.name, b)
    print(f"\n[{run.name}] mutual matches: {[len(x) for x in lists]}")


def test_crop_margin_is_never_read():
    """A 727 x 545 batch whose 13-pixel margins are NaN gives, bit for bit, what the 714 x 532 crop of the same pixels
    gives: every output of compute_matches and the solver's pose, sampled sets and inlier mask, none of them NaN."""
    variant, B, H, W, im, ir, _ = st.GEOMETRIES["crop"]
    cfg = mickey_cfg(variant, im, ir)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
    model = model.cuda().eval()
    Hc, Wc = H // 14 * 14, W // 14 * 14
    full = synthetic_pair(B, H, W, seed=17)
    for k in ("image0", "image1"):
        full[k][:, :, Hc:] = float("nan")
        full[k][:, :, :, Wc:] = float("nan")
    full = {k: v.to(DEV) for k, v in full.items()}
    crop = {k: (v[:, :, :Hc, :Wc].contiguous() if k.startswith("image") else v.clone()) for k, v in full.items()}
    outs = []
    for data in (full, crop):
        with torch.no_grad():
            model.compute_matches(data)
            data["final_scores"] = data.pop("_final_scores_fused")
            model.e2e_Procrustes.estimate_pose_vectorized(data, seed=st.SEED)
        torch.cuda.synchronize()
        res = data.pop("_solver")
        outs.append({**{k: v for k, v in data.items() if torch.is_tensor(v) and not k.startswith("image")},
                     **{k: v for k, v in res.items() if v is not None}})
    a, b = outs
    assert set(a) == set(b) and {"kps0", "dsc1", "scores", "final_scores", "pose", "sampled_idx", "inlier_mask"} <= set(a)
    for k in a:
        assert torch.equal(a[k], b[k]), k
        if a[k].is_floating_point():
            assert not bool(torch.isnan(a[k]).any()), k
