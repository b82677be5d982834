"""CPU checks of the training loss: the oracle (oracle/loss_oracle.py) against the live reference's recorded outputs
(tests/golden/reference_loss_small.npz), the VCRE grid, which inner draws torch.multinomial refuses, and the host-side
argument checks of mk_loss_search / mk_loss_gradient."""
import ctypes as C

import numpy as np
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.loss import LossParams, MetricPoseLoss, vcre_grid
from oracle import loss_oracle as lo
from tests import loss_cases

FIX = np.load(loss_cases.FIXTURE)
FIX_WARMUP = np.load(loss_cases.WARMUP_FIXTURE)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("name", list(loss_cases.CASES))
def test_oracle_matches_reference_fixture(name):
    """With the reference's two draws injected, the fp32 oracle reproduces every recorded output: the final inlier mask
    of every hypothesis exactly, scores / losses / baseline / avg_loss to 1e-5 relative, the REINFORCE gradient on the
    same support to 1e-5, and the kps / depth gradients of avg_loss.backward() to 1e-4 (torch's SVD backward
    amplifies the fp32 rounding of near-degenerate 8-point hypotheses)."""
    _oracle_reproduces(FIX, name)


@pytest.mark.parametrize("name", list(loss_cases.WARMUP_CASES))
def test_oracle_matches_reference_warmup_fixture(name):
    """The same, under the reference's two warm-up configs: 64 samples per set, no null hypothesis, top-K at B = 4."""
    assert LossParams(loss_cases.case_cfg(name)).n_sample == 64
    _oracle_reproduces(FIX_WARMUP, name)


def _oracle_reproduces(FIX, name):
    p = f"{name}/"
    batch = loss_cases.case_batch(name)
    prm = LossParams(loss_cases.case_cfg(name))
    r = lo.metric_pose_loss(batch, prm, outer_idx=torch.from_numpy(FIX[p + "outer_idx"]).long(),
                            inner_idx=torch.from_numpy(FIX[p + "inner_idx"]).long(), dtype=torch.float32)
    assert r["num_valid_h"] == int(FIX[p + "num_valid_h"]) == 1
    inl = np.unpackbits(FIX[p + "inliers_final"], axis=1, bitorder="little")[:, :prm.n_sample]
    assert np.array_equal(r["inliers_final"].numpy().astype(np.uint8), inl)
    assert _rel(r["scores"].detach(), FIX[p + "scores"]) < 1e-5
    assert _rel(r["loss_value"].detach(), FIX[p + "loss_value"]) < 1e-5
    assert _rel(r["baseline"].detach(), FIX[p + "baseline"]) < 1e-5
    assert _rel(r["avg_loss"].detach(), FIX[p + "avg_loss"]) < 1e-5
    assert np.array_equal(r["mask_topk"].numpy(), FIX[p + "mask_topk"])
    g = r["probs_grad"].reshape(-1)
    nz = torch.nonzero(g).reshape(-1).numpy()
    assert np.array_equal(nz, FIX[p + "grad_idx"])
    assert _rel(g[nz], FIX[p + "grad_val"]) < 1e-5
    r["avg_loss"].backward()
    for k in ("kps0", "kps1", "depth0", "depth1"):
        assert _rel(r[k].grad, FIX[p + k + "_grad"]) < 1e-4, k


def test_vcre_grid_regenerated_from_its_definition():
    assert np.array_equal(vcre_grid().numpy(), FIX["vcre_grid"])


@pytest.mark.parametrize("positive", [0, 1, 7, 8, 512])
def test_inner_draw_raise_table(positive):
    """torch.multinomial(weights, 8) without replacement over a 512-entry set raises only when the set's scores sum to
    zero; with 1 to 7 positive scores it fills the draw with zero-score entries.  mk_loss_search sets
    MK_LOSS_STATUS_INNER exactly for the first case (the GPU tests hold it to this table)."""
    w = torch.zeros(1, 512)
    w[0, torch.randperm(512, generator=torch.Generator().manual_seed(positive))[:positive]] = 0.5
    raised = False
    try:
        torch.multinomial(w, 8)
    except RuntimeError:
        raised = True
    assert raised == (positive == 0)


def test_loss_params_follow_the_released_config():
    p = LossParams(loss_cases.loss_cfg(it_matches=20, it_ransac=20, topk=True))
    assert (p.n_sample, p.num_corr, p.num_ref_steps, p.it_matches, p.it_ransac) == (512, 8, 4, 20, 20)
    assert (p.inlier_3d_th, p.inlier_ref_th, p.score_temperature, p.max_loss_null) == (0.3, 0.15, 20.0, 0.8)
    assert p.train_w_top and p.topK == 30
    cfg = loss_cases.loss_cfg()
    cfg.LOSS_CLASS.LOSS_FUNCTION = "L2"
    with pytest.raises(ValueError):
        LossParams(cfg)


# reference config -> (n_sample, num_corr, num_ref_steps, it_matches, it_ransac, add_null_hypothesis, train_w_top, topK,
#                      loss_type, soft_clipping, inlier_3d_th, inlier_ref_th, score_temperature, max_loss_null, th_outliers)
REFERENCE_LOSS_PARAMS = {
    "curriculum_learning": (512, 8, 4, 20, 20, True, True, 30, "VCRE", True, 0.3, 0.15, 20.0, 0.8, 0.35),
    "overlap_score": (512, 8, 4, 20, 20, True, False, None, "VCRE", True, 0.3, 0.15, 20.0, 0.8, 0.35),
    "curriculum_learning_warm_up": (64, 8, 4, 20, 20, False, True, 30, "VCRE", True, 0.3, 0.15, 20.0, 0.8, 0.35),
    "overlap_score_warm_up": (64, 8, 4, 20, 20, False, False, None, "VCRE", True, 0.3, 0.15, 20.0, 0.8, 0.35),
}


@pytest.mark.parametrize("name", list(REFERENCE_LOSS_PARAMS))
def test_loss_params_read_every_reference_config(name):
    """All four configs the reference ships, as its dump of them reads: MetricPoseLoss accepts each one."""
    p = LossParams(loss_cases.reference_cfg(name))
    got = (p.n_sample, p.num_corr, p.num_ref_steps, p.it_matches, p.it_ransac, p.add_null_hypothesis, p.train_w_top,
           p.topK, p.loss_type, p.soft_clipping, p.inlier_3d_th, p.inlier_ref_th, p.score_temperature, p.max_loss_null,
           p.th_outliers)
    assert got == REFERENCE_LOSS_PARAMS[name]


@pytest.mark.parametrize("key,value", [("NUM_SAMPLES_MATCHES", 48), ("NUM_SAMPLES_MATCHES", 4096),
                                       ("NUM_SAMPLES_MATCHES", 0), ("NUM_SAMPLES_MATCHES", 500),
                                       ("NUM_CORR_3d3d", 17), ("NUM_CORR_3d3d", 0)])
def test_loss_params_reject_unsupported_sizes(key, value):
    """A set size that is not a multiple of 32 up to 2048, or more than 16 (or no) correspondences per hypothesis, fails
    at construction rather than at the first forward."""
    cfg = loss_cases.reference_cfg("curriculum_learning_warm_up")
    lc = cfg.LOSS_CLASS
    if key == "NUM_SAMPLES_MATCHES":
        lc.SAMPLER.NUM_SAMPLES_MATCHES = value
    else:
        lc.GENERATE_HYPOTHESES.NUM_CORR_3d3d = value
    with pytest.raises(ValueError, match=key):
        LossParams(cfg)
    with pytest.raises(ValueError, match=key):
        MetricPoseLoss(cfg)


def test_metric_pose_loss_rejects_cpu_tensors():
    with pytest.raises(ValueError):
        MetricPoseLoss(loss_cases.case_cfg("vits_vcre"))(loss_cases.case_batch("vits_vcre"))


def _search(lib, B=2, N=64, IM=4, IR=8, S=512, Cn=8, n_ref=4, th=0.15, pitch=0, ws_bytes=None, null=None):
    fake = C.c_void_p(0x10000)
    ptrs = [fake] * 15
    if null is not None:
        ptrs[null] = None
    fs, k0, d0, k1, d1, K0, K1, oi, ii, so, io, bo, st, ws = ptrs[:14]
    if ws_bytes is None:
        ws_bytes = lib.mk_loss_search_ws_bytes(B, IM)
    return lib.mk_loss_search(fs, pitch, k0, d0, k1, d1, K0, K1, B, N, IM, IR, S, Cn, n_ref, th, 1, oi, ii, so, io, bo, st,
                              ws, ws_bytes, None)


def test_search_rejects_bad_arguments_before_launching():
    """Every rejected call returns MK_ERR_INVALID from the host checks (the pointers are never dereferenced)."""
    lib = _lib.load()
    bad = [dict(B=0), dict(N=0), dict(IM=0), dict(IR=0), dict(S=500), dict(S=4096), dict(S=0), dict(Cn=0), dict(Cn=17),
           dict(S=48), dict(S=16), dict(S=2080), dict(S=32, Cn=33), dict(S=64, Cn=17), dict(S=64, N=7),
           dict(n_ref=-1), dict(th=float("nan")), dict(N=20), dict(pitch=10), dict(N=50000), dict(ws_bytes=16),
           dict(null=0), dict(null=3), dict(null=6), dict(null=9), dict(null=11), dict(null=12), dict(null=13)]
    for kw in bad:
        assert _search(lib, **kw) == -1, kw
        assert b"mk_loss_search" in lib.mk_last_error(), kw


@pytest.mark.parametrize("S", [32, 64, 96, 288, 512, 2048])
def test_search_accepts_every_multiple_of_32(S):
    """Every set size that is a multiple of 32 up to 2048 passes the argument check: with a short workspace the call
    stops at the workspace check instead (the pointers are never dereferenced)."""
    lib = _lib.load()
    assert _search(lib, S=S, ws_bytes=16) == -1
    assert b"mk_loss_search: workspace of 16 bytes" in lib.mk_last_error()


def test_gradient_rejects_bad_arguments_before_launching():
    lib = _lib.load()
    fake = C.c_void_p(0x10000)

    def call(B=2, N=64, IM=4, S=512, ws_bytes=None, null=None):
        p = [fake] * 6
        if null is not None:
            p[null] = None
        ws_bytes = lib.mk_loss_gradient_ws_bytes(B, IM, S) if ws_bytes is None else ws_bytes
        return lib.mk_loss_gradient(p[0], p[1], p[2], p[3], B, N, IM, S, p[4], p[5], ws_bytes, None)

    for kw in [dict(B=0), dict(N=0), dict(IM=0), dict(S=0), dict(S=4096), dict(N=50000), dict(ws_bytes=4)] + \
              [dict(null=i) for i in range(6)]:
        assert call(**kw) == -1, kw
        assert b"mk_loss_gradient" in lib.mk_last_error(), kw
