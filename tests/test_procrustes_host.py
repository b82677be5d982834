"""The handle-free pose solver without a GPU: the drop-in e2eProbabilisticProcrustesSolver's attributes and configuration
checks (NUM_SAMPLED_MATCHES = 2048 only, as the live reference's zero result below 2048 shows), mk_procrustes_solve's
host-side rejections (the pointers are never dereferenced), and
use_cuda_modules(model, solver=True) on the recorded training-model tree and, when the reference tree is present, on the
live MicKeyTrainingModel."""
import ctypes as C
import sys

import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.model import MickeyRelativePose
from mickey_b200.procrustes import e2eProbabilisticProcrustesSolver
from mickey_b200.training import use_cuda_modules
from oracle import mickey_oracle as mo
from oracle import ref_harness
from tests import planted
from tests.common import rotation_angle_deg
from tests.golden import make_training_tree as mtt
from tests.test_heads_host import model_from_tree, needs_reference

ATTRS = {"it_RANSAC": "IT_RANSAC", "it_matches": "IT_MATCHES", "num_samples_matches": "NUM_SAMPLED_MATCHES",
         "num_corr_3d_3d": "NUM_CORR_3D_3D", "num_refinements": "NUM_REFINEMENTS", "th_inlier": "TH_INLIER",
         "th_soft_inlier": "TH_SOFT_INLIER"}       # probabilisticProcrustes.py:11-19


class ReferenceSolverStandIn:
    """What the reference's e2eProbabilisticProcrustesSolver.__init__ (probabilisticProcrustes.py:11-19) holds: the
    recorded tree has no solver, so this stands in for it."""

    def __init__(self, cfg):
        for attr, key in ATTRS.items():
            setattr(self, attr, cfg.PROCRUSTES[key])


def attrs(solver):
    return {a: getattr(solver, a) for a in ATTRS}


@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_attributes_are_the_reference_classes(config):
    cfg = mtt.training_cfg(config)
    ours = e2eProbabilisticProcrustesSolver(cfg)
    assert attrs(ours) == attrs(ReferenceSolverStandIn(cfg))
    assert attrs(ours) == dict(it_RANSAC=100, it_matches=20, num_samples_matches=2048, num_corr_3d_3d=3,
                               num_refinements=4, th_inlier=0.15, th_soft_inlier=0.3)


@needs_reference
@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_attributes_are_the_live_reference_classes(config):
    model = mtt.reference_training_model(mtt.training_cfg(config), variant="vits")
    assert attrs(e2eProbabilisticProcrustesSolver(model.cfg)) == attrs(model.e2e_Procrustes)


UNSUPPORTED = {"IT_MATCHES": [0, 65536], "IT_RANSAC": [0, 2 ** 31 // 20 + 1], "NUM_SAMPLED_MATCHES": [0, 100, 255, 2304, 4096],
               "NUM_CORR_3D_3D": [2, 4], "NUM_REFINEMENTS": [-1], "TH_INLIER": [0.0, -0.1, float("nan"), float("inf")],
               "TH_SOFT_INLIER": [0.0, float("nan")]}


@pytest.mark.parametrize("key,value", [(k, v) for k, vs in UNSUPPORTED.items() for v in vs])
def test_unsupported_configurations_raise_at_construction(key, value):
    cfg = mtt.training_cfg()
    cfg.PROCRUSTES[key] = value
    with pytest.raises(ValueError, match=key):
        e2eProbabilisticProcrustesSolver(cfg)


@pytest.mark.parametrize("S", [256, 512, 1024, 1536, 1792])
def test_set_sizes_the_reference_cannot_run_raise_at_construction(S):
    """Multiples of 256 below 2048 are inside mk_procrustes_solve's range (tests/test_gpu_solver_params.py runs them),
    but the reference returns the zero pose for every one of them (test_reference_returns_the_zero_pose_below_2048):
    both drop-ins reject them, naming the reference's lines."""
    cfg = mtt.training_cfg()
    cfg.PROCRUSTES.NUM_SAMPLED_MATCHES = S
    with pytest.raises(ValueError, match=r"NUM_SAMPLED_MATCHES must be 2048.*probabilisticProcrustes\.py:271-272"):
        e2eProbabilisticProcrustesSolver(cfg)
    icfg = mickey_cfg("vits")
    icfg.PROCRUSTES.NUM_SAMPLED_MATCHES = S
    with pytest.raises(ValueError, match=r"NUM_SAMPLED_MATCHES must be 2048.*probabilisticProcrustes\.py:271-272"):
        MickeyRelativePose(icfg)
    assert MickeyRelativePose(mickey_cfg("vits")).e2e_Procrustes.num_samples_matches == 2048


def _reference_solver_class():
    ref_harness._install_stubs()
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    try:
        with ref_harness._ref_on_path():
            from lib.models.MicKey.modules.utils.probabilisticProcrustes import e2eProbabilisticProcrustesSolver as Ref
    finally:
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return Ref


@needs_reference
def test_reference_returns_the_zero_pose_below_2048():
    """The live reference's estimate_pose_vectorized on a planted problem: a real pose at NUM_SAMPLED_MATCHES = 2048,
    the zero result at 512 (its reshape to 2048 samples per set raises inside its try, :271-272), where the fp64
    oracle, which stays general, returns the planted pose."""
    Ref = _reference_solver_class()
    p = planted.planted_problem((20, 16), batch=2, seed=5)
    batch = {"final_scores": p["final_scores"], "kps0": p["kps0"], "kps1": p["kps1"], "depth_kp0": p["depth0"],
             "depth_kp1": p["depth1"], "K_color0": p["K"], "K_color1": p["K"]}
    cfg = mickey_cfg("vits", 2, 8)
    torch.manual_seed(0)
    R, t, inl = Ref(cfg).estimate_pose_vectorized(dict(batch))
    assert float(R.abs().max()) > 0.5 and float(inl.abs().max()) > 0
    cfg.PROCRUSTES.NUM_SAMPLED_MATCHES = 512
    torch.manual_seed(0)
    R, t, inl, lst = Ref(cfg).estimate_pose_vectorized(dict(batch), return_inliers=True)
    assert torch.equal(R, torch.zeros(2, 3, 3)) and torch.equal(t, torch.zeros(2, 1, 3)) and torch.equal(inl, torch.zeros(2))
    assert len(lst) == 2 and all(x.shape == (0, 5) for x in lst)
    Ro, to, _ = mo.solve_pose(*(batch[k].double() for k in ("final_scores", "kps0", "depth_kp0", "kps1", "depth_kp1",
                                                            "K_color0", "K_color1")), cfg,
                              generator=torch.Generator().manual_seed(0))
    assert float(rotation_angle_deg(Ro, p["R"].double()).max()) < 0.1            # fp32 keypoints: not exact
    assert float((to.reshape(2, 3) - p["t"].double().reshape(2, 3)).abs().max()) < 1e-2


# ---- mk_procrustes_solve's host checks ------------------------------------------------------------------------------
GOOD = dict(B=8, N=1938, IM=20, IR=100, S=2048, Cn=3, n_ref=4, th=0.15, th_soft=0.3, pitch=1938)


def _solve(lib, ws_bytes=None, null=None, **kw):
    a = dict(GOOD, **kw)
    fake = C.c_void_p(0x10000)
    p = [fake] * 14        # final_scores, kps, depth, K0, K1, outer, inner, pose, best_set, mask, sampled, hyp, status, ws
    p[5] = p[6] = None
    if null is not None:
        p[null] = None
    if ws_bytes is None:
        ws_bytes = max(lib.mk_procrustes_ws_bytes(a["B"], a["N"], a["IM"], a["IR"], a["S"]), 1 << 30)
    return lib.mk_procrustes_solve(p[0], a["pitch"], p[1], p[2], p[3], p[4], a["B"], a["N"], a["IM"], a["IR"], a["S"],
                                   a["Cn"], a["n_ref"], a["th"], a["th_soft"], 1, p[5], p[6], p[7], p[8], p[9], p[10],
                                   p[11], p[12], p[13], ws_bytes, None)


BAD = [dict(B=0), dict(B=65536), dict(N=0), dict(N=46341, pitch=46341), dict(IM=0), dict(IM=65536), dict(IR=0),
       dict(IM=30000, IR=100000), dict(B=65535, IM=65535), dict(S=0), dict(S=100), dict(S=2304), dict(S=4096),
       dict(Cn=2), dict(Cn=4), dict(n_ref=-1), dict(th=0.0), dict(th=float("nan")), dict(th=float("inf")),
       dict(th_soft=-1.0), dict(th_soft=float("nan")), dict(pitch=1937), dict(ws_bytes=16)] + \
      [dict(null=i) for i in (0, 1, 2, 3, 4, 7, 13)]


@pytest.mark.parametrize("kw", BAD, ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()))
def test_solve_rejects_bad_arguments_before_launching(kw):
    """Every rejected call returns MK_ERR_INVALID with a message from the host checks; nothing is launched (on a machine
    without a GPU a launch would return MK_ERR_CUDA instead)."""
    lib = _lib.load()
    assert _solve(lib, **kw) == -1
    assert b"mk_procrustes_solve" in lib.mk_last_error()


def test_workspace_size_of_the_validation_shapes_and_of_bad_sizes():
    lib = _lib.load()
    for B, N in ((8, 1938), (24, 850)):
        nbytes = lib.mk_procrustes_ws_bytes(B, N, 20, 100, 2048)
        assert 0 < nbytes < B * (2 << 20) and nbytes % 256 == 0        # under 2 MB per pair
        # the solver's scratch: 2048 drawn cells per stream, score and [R | t] per hypothesis, and the sampler's
        # 8192 candidates per stream dominate
        assert nbytes >= B * 20 * (2048 * 4 + 100 * 13 * 4 + 8192 * 8)
        assert _solve(lib, B=B, N=N, pitch=N, ws_bytes=nbytes - 1) == -1
        assert b"workspace of" in lib.mk_last_error()
    for bad in ((0, 1938, 20, 100, 2048), (8, 0, 20, 100, 2048), (8, 1938, 20, 100, 300), (8, 1938, 0, 100, 2048)):
        assert lib.mk_procrustes_ws_bytes(*bad) == -1


@pytest.mark.parametrize("S", [256, 1024, 2048])
def test_supported_sizes_pass_the_argument_checks(S):
    """With a short workspace a supported call stops at the workspace check: every earlier check accepted it."""
    lib = _lib.load()
    assert _solve(lib, S=S, ws_bytes=16) == -1
    assert b"mk_procrustes_solve: workspace of 16 bytes" in lib.mk_last_error()


# ---- use_cuda_modules(model, solver=True) -----------------------------------------------------------------------------
def snapshot(model):
    return {n: (t, t.detach().clone()) for n, t in model.state_dict(keep_vars=True).items()}


def assert_same_state(model, before):
    after = model.state_dict(keep_vars=True)
    assert list(after) == list(before)
    assert all(after[n] is t and torch.equal(t, v) for n, (t, v) in before.items())


def check_solver_swap(model):
    old = model.e2e_Procrustes
    use_cuda_modules(model)
    assert model.e2e_Procrustes is old                               # solver=False: the reference's solver stays
    before = snapshot(model)
    mods = dict(model.named_modules())
    assert use_cuda_modules(model, solver=True) is model
    new = model.e2e_Procrustes
    assert type(new) is e2eProbabilisticProcrustesSolver and attrs(new) == attrs(old)
    assert_same_state(model, before)
    assert dict(model.named_modules()) == mods
    use_cuda_modules(model, solver=True)                             # a second call changes nothing
    assert model.e2e_Procrustes is new
    assert_same_state(model, before)


def check_solver_rejected(model):
    old = model.e2e_Procrustes
    before = snapshot(model)
    mods = dict(model.named_modules())
    model.cfg.PROCRUSTES.NUM_SAMPLED_MATCHES = 100
    with pytest.raises(ValueError, match="NUM_SAMPLED_MATCHES"):
        use_cuda_modules(model, solver=True)
    assert model.e2e_Procrustes is old
    assert dict(model.named_modules()) == mods                       # no module was swapped either
    assert_same_state(model, before)


def tree_with_solver(config="curriculum_learning"):
    model = model_from_tree(config)
    model.e2e_Procrustes = ReferenceSolverStandIn(model.cfg)
    return model


@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_use_cuda_modules_swaps_the_solver_of_the_recorded_tree(config):
    check_solver_swap(tree_with_solver(config))


def test_use_cuda_modules_rejects_a_solver_config_without_touching_the_recorded_tree():
    check_solver_rejected(tree_with_solver())


@needs_reference
@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_use_cuda_modules_swaps_the_solver_of_the_live_reference_model(config):
    check_solver_swap(mtt.reference_training_model(mtt.training_cfg(config), variant="vits"))


@needs_reference
def test_use_cuda_modules_rejects_a_solver_config_without_touching_the_live_reference_model():
    check_solver_rejected(mtt.reference_training_model(mtt.training_cfg(), variant="vits"))
