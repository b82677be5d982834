"""Every kernel stage, the solver's draws and the mutual matches under the configuration branches the released YAML does
not take, element by element against fp64.

The head and matcher flags the engine reads (engine.py make_mk_config) select arithmetic inside the kernels:
KP_HEADS.USE_SOFTMAX (score_activation_kernel: sigmoid x border), USE_DEPTHSIGMOID (kp_head_out_kernel: MAX_DEPTH
sigma), FEATURE_MATCHER.DUAL_SOFTMAX.USE_DUSTBIN (matcher_lse_reduce without the dustbin), the two POS_ENCODING flags
(rb3 conv2's aux_group_mask 0x7 / 0x8), DSC_HEAD.NORM_DSC (desc_out_kernel without normalisation) and TEMPERATURE (the
matcher's fixed-shift partials for unit-norm descriptors while 1 / T <= 25, true maxima otherwise).  tests/stages.py
builds the fp64 reference of the branch each run's config takes, with a planted mutation per branch (the border dropped
from the sigmoid score, MAX_DEPTH dropped, the dustbin included when off, normalisation applied when off, the PE on a
group whose flag is off) that its bound must reject.  `max(err / bound)` per stage goes to $MICKEY_STAGE_METRICS.
"""
import pytest
import torch

from oracle.matches_oracle import matches_list
from tests import elementwise as ew
from tests import stages as st

pytestmark = pytest.mark.gpu

SOFTMAX = "MICKEY.KP_HEADS.USE_SOFTMAX"
DEPTH_SIGMOID = "MICKEY.KP_HEADS.USE_DEPTHSIGMOID"
DUSTBIN = "FEATURE_MATCHER.DUAL_SOFTMAX.USE_DUSTBIN"
KP_PE, DSC_PE = "MICKEY.KP_HEADS.POS_ENCODING", "MICKEY.DSC_HEAD.POS_ENCODING"
NORM_DSC = "MICKEY.DSC_HEAD.NORM_DSC"
TEMP = "FEATURE_MATCHER.DUAL_SOFTMAX.TEMPERATURE"
ALL_FLIPPED = {SOFTMAX: False, DEPTH_SIGMOID: True, DUSTBIN: False, KP_PE: False, DSC_PE: False, NORM_DSC: False, TEMP: 1.0}

C2 = ("vits", 1, 720, 540, 8, 64, "one tile")
# id -> (overrides, (variant, B, H, W, IM, IR, GEMM regime of the relaunches))
CASES = {
    "sigmoid_scores": ({SOFTMAX: False}, C2),
    "depth_sigmoid": ({DEPTH_SIGMOID: True}, C2),
    "no_dustbin": ({DUSTBIN: False}, C2),
    "no_dustbin_t1": ({DUSTBIN: False, TEMP: 1.0}, C2),    # unit-norm at T = 1: the dustbin's share is resolvable
    "pe_kp_only": ({KP_PE: True, DSC_PE: False}, C2),
    "pe_dsc_only": ({KP_PE: False, DSC_PE: True}, C2),
    "pe_none": ({KP_PE: False, DSC_PE: False}, C2),
    "raw_dsc_t20": ({NORM_DSC: False, TEMP: 20.0}, C2),
    "raw_dsc_t1": ({NORM_DSC: False, TEMP: 1.0}, C2),
    "cold_t002": ({TEMP: 0.02}, C2),                    # unit-norm, 1 / T = 50: true maxima
    "edge_t004": ({TEMP: 0.04}, C2),                    # unit-norm, 1 / T = 25: the last fixed-shift temperature
    "all_flipped_c3": (ALL_FLIPPED, ("vitb", 8, 720, 540, 16, 64, "persistent")),
    "all_flipped_min": (ALL_FLIPPED, ("vits", 1, 98, 98, 8, 64, "one tile")),
}


@pytest.fixture(scope="module", params=list(CASES))
def run(request):
    overrides, geo = CASES[request.param]
    r = st.Run(request.param, *geo, overrides=overrides)
    yield r
    del r
    torch.cuda.empty_cache()


def test_config_reaches_the_engine(run):
    """The handle holds the run's flags, and the C3-sized run's matcher GEMM reaches the persistent kernel: EPI_LSE
    over B * 16 * 16 = 2048 tiles, more than 8 per SM (EPI_DUAL runs the same grid one tile per CTA)."""
    c = run.eng.mkcfg
    assert (bool(c.use_softmax), bool(c.depth_sigmoid), bool(c.use_dustbin), bool(c.norm_dsc)) == \
        (run.use_softmax, run.depth_sigmoid, run.use_dustbin, run.norm_dsc)
    assert (bool(c.kp_pos_enc), bool(c.dsc_pos_enc)) == (bool(run.cfg.MICKEY.KP_HEADS.POS_ENCODING),
                                                         bool(run.cfg.MICKEY.DSC_HEAD.POS_ENCODING))
    assert abs(c.temperature - run.temperature) <= 1e-7 * run.temperature
    lse = ew.GemmTiles(run.N, run.npad, run.B, sms=run.sms)
    assert lse.persistent == (run.name == "all_flipped_c3"), (run.name, lse.tiles)


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
    """The outer draws against the fp64 race, the inner triples bit for bit, the hypotheses against fp64.  The outer draw
    alone at 98 x 98, where the matrix has one positive cell and its Kabsch problems are degenerate
    (tests/test_gpu_stages_geometries.py), and with raw descriptors, whose logits of hundreds put the synthetic
    final_scores on a few cells: most triples are then degenerate and the hypothesis scores tie within their bound."""
    sol = st.Solved(run.name, run.cfg, run.model, run.data, run.B, run.im, run.ir)
    st.outer_draws_are_the_race(sol)
    if run.N > 49 and run.norm_dsc:
        st.inner_draws_are_restated(sol)


def test_mutual_matches(run):
    """model.mutual_matches on the run's final_scores equals the oracle exactly."""
    fs = run.data["_final_scores_fused"]
    lists, scores = run.model.mutual_matches(fs)
    for b in range(run.B):
        rm, rv = matches_list(fs[b].cpu())
        assert torch.equal(lists[b].cpu(), rm) and torch.equal(scores[b].cpu(), rv), (run.name, b)
    print(f"\n[{run.name}] mutual matches: {[len(x) for x in lists]}")
