"""Grading Map-free submissions without a GPU: the fp64 oracle against the benchmark's recorded per-frame values, the pose
parser against the benchmark's, mk_mapfree_frame_metrics's host-side rejections (the pointers are never dereferenced),
and whole submissions through mapfree_eval's evaluator and CLI with the oracle in the kernel's place."""
import ctypes as C
import json
import logging
import os
import sys
from io import StringIO
from pathlib import Path

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "compat")) if __import__("importlib").util.find_spec("transforms3d") is None else None

from mickey_b200 import _lib  # noqa: E402
from mickey_b200 import mapfree_eval as mfe  # noqa: E402
from oracle import mapfree_eval_oracle as orc  # noqa: E402
from tests import mapfree_fixture as mf  # noqa: E402

FIX = mf.FIX


@pytest.fixture
def tree(tmp_path):
    return mf.write_tree(tmp_path)


@pytest.fixture
def oracle_kernel(monkeypatch):
    """The evaluator's per-frame errors come from the oracle instead of the kernel."""
    monkeypatch.setattr(mfe, "frame_metrics", orc.frame_metrics)


def close(a, b, rel=1e-12):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all(np.abs(a - b) <= rel * np.abs(b)))


# ---- the oracle against the benchmark ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", mf.GRADED_ZIPS)
def test_oracle_reproduces_every_per_frame_value(tree, name):
    for scene, fr in mf.graded_frames(tree, name):
        got = orc.frame_metrics(fr["q_est"], fr["t_est"], fr["q_gt"], fr["t_gt"], fr["K"], fr["W"], fr["H"])
        assert close(got, mf.reference_values(name, scene)), (name, scene)


def test_the_crafted_submissions_cover_their_cases(tree):
    allv = {z: np.concatenate([mf.reference_values(z, s) for s, _ in mf.graded_frames(tree, z)]) for z in mf.GRADED_ZIPS}
    assert allv["near_perfect"][:, 2].max() < 10 and allv["near_perfect"][:, 1].max() < 1
    assert allv["large_errors"][:, 0].min() > 0.5
    assert 179 < allv["near_180"][:, 1].min() and np.isfinite(allv["near_180"]).all()
    # grid points behind the estimate's camera: a negative depth in the residual transform
    behind = 0
    for _, fr in mf.graded_frames(tree, "behind_camera"):
        for i in range(len(fr["confidence"])):
            qe, ce = orc.world2cam_to_cam2world(fr["q_est"][i], fr["t_est"][i])
            qg, cg = orc.world2cam_to_cam2world(fr["q_gt"][i], fr["t_gt"][i])
            E, G = np.eye(4), np.eye(4)
            E[:3, :3], E[:3, 3], G[:3, :3], G[:3, 3] = orc.quat2mat(qe), ce, orc.quat2mat(qg), cg
            behind += int(((np.linalg.inv(E) @ G @ orc._EYE.T)[2] < 0).any())
    assert behind >= 10
    norms = np.concatenate([np.linalg.norm(fr["q_est"], axis=1) for _, fr in mf.graded_frames(tree, "nonunit_quaternions")])
    assert norms.min() < 0.6 and norms.max() > 2.5
    conf = [c for _, fr in mf.graded_frames(tree, "confidence_ties") for c in fr["confidence"]]
    assert 0.0 in conf and len(set(conf)) < len(conf) / 4
    assert {fr["W"] for z in mf.GRADED_ZIPS for _, fr in mf.graded_frames(tree, z)} == {540.0, 960.0}
    rec = FIX["zips"]["malformed_and_missing"]
    assert rec["scenes"]["s00003"] == {"failures": 16, "results": {}}           # missing scene: failures before subsampling
    assert rec["scenes"]["s00000"]["failures"] == 3                              # frames 5, 15 and 25


# ---- the pose parser -------------------------------------------------------------------------------------------------------
def parsed_rows(text, name, conf):
    f = StringIO(text)
    f.name = name
    out = []
    for frame, (q, t, c) in mfe.load_poses(f, load_confidence=conf).items():
        qi, ti = orc.world2cam_to_cam2world(q, t)                 # the benchmark's parser hands them over camera-to-world
        out.append([frame, list(qi), list(ti)] + ([c] if conf else []))
    return out


def assert_same_rows(ours, ref):
    assert [r[0] for r in ours] == [r[0] for r in ref]
    for a, b in zip(ours, ref):
        assert close(a[1], b[1], 1e-15) and close(a[2], b[2], 1e-15)
        assert a[3:] == b[3:]


@pytest.mark.parametrize("name", list(FIX["zips"]))
def test_load_poses_parses_every_crafted_line_as_the_benchmark(name):
    for member, text in FIX["zips"][name]["files"].items():
        assert_same_rows(parsed_rows(text, member, True), FIX["zips"][name]["parsed"][member])


def test_load_poses_parses_the_ground_truth_as_the_benchmark():
    for scene, files in FIX["scenes"].items():
        assert_same_rows(parsed_rows(files["poses.txt"], "poses.txt", False), FIX["gt_parsed"][scene])


def test_load_poses_rules():
    text = "\n".join(["a/frame_00003.jpg 1 0 0 0 1 2 3 7",
                      "a/frame_00004.jpg 1 0 0 0 1 2 3",                    # wrong field count
                      "#a/frame_00005.jpg 1 0 0 0 1 2 3 7",                 # comment
                      "a/frame_0000x.jpg 1 0 0 0 1 2 3 7",                  # no frame number
                      "a/frame_00006.jpg 1 0 0 nan 1 2 3 7",                # NaN
                      "a/frame_00007.jpg 1 0 0 0 1 2 3 -inf",               # infinite
                      "a/frame_00008.jpg 1e-9 0 0 0 1 2 3 7",               # norm close to zero
                      "a/frame_00009.jpg 2 0 0 0 1 2 3 0",
                      "a/frame_00003.jpg 0 1 0 0 4 5 6 8"])                 # replaces frame 3, keeps its place
    poses = mfe.load_poses(StringIO(text), load_confidence=True)
    assert list(poses) == [3, 9]
    q, t, c = poses[3]
    assert list(q) == [0, 1, 0, 0] and list(t) == [4, 5, 6] and c == 8.0
    assert list(poses[9][0]) == [2, 0, 0, 0] and poses[9][2] == 0.0
    assert list(mfe.subsample_poses({k: k for k in (4, 9, 1, 7, 3, 2, 8)}, 3)) == [4, 7, 8]


# ---- mk_mapfree_frame_metrics's host checks ------------------------------------------------------------------------------
def _metrics(lib, P=100, W=540, H=720, null=None):
    p = [C.c_void_p(0x10000)] * 7             # q_est, t_est, q_gt, t_gt, K, grid, err
    if null is not None:
        p = list(p)
        p[null] = None
    return lib.mk_mapfree_frame_metrics(*p[:6], P, W, H, p[6], None)


MAX_FRAMES = 67108863
BAD = [dict(P=0), dict(P=-1), dict(P=MAX_FRAMES + 1), dict(P=2 ** 31 - 1), dict(W=0), dict(H=0), dict(W=-540),
       dict(H=-1)] + [dict(null=i) for i in range(7)]


@pytest.mark.parametrize("kw", BAD, ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()))
def test_frame_metrics_rejects_bad_arguments_before_launching(kw):
    """Every rejected call returns MK_ERR_INVALID with a message from the host checks; nothing is launched (on a machine
    without a GPU a launch would return MK_ERR_CUDA instead)."""
    lib = _lib.load()
    assert _metrics(lib, **kw) == -1
    assert b"mk_mapfree_frame_metrics" in lib.mk_last_error()


def test_the_frame_limit_is_the_headers():
    header = open(os.path.join(ROOT, "include", "mickey_b200.h")).read()
    assert f"#define MK_MAPFREE_MAX_FRAMES {MAX_FRAMES}" in header and MAX_FRAMES * 32 < 2 ** 31 <= (MAX_FRAMES + 1) * 32
    assert "#define MK_VCRE_POINTS 196" in header


def test_the_python_wrapper_rejects_bad_tensors_before_the_library():
    import torch
    q, t, K = torch.zeros(2, 4, dtype=torch.float64), torch.zeros(2, 3, dtype=torch.float64), torch.zeros(2, 3, 3)
    with pytest.raises(ValueError, match="K"):
        mfe.frame_metrics_dev(q, t, q, t, K, 540, 720)
    with pytest.raises(ValueError, match="CUDA"):
        mfe.frame_metrics_dev(q, t, q, t, K.double(), 540, 720)


# ---- whole submissions, with the oracle in the kernel's place ---------------------------------------------------------------
@pytest.mark.parametrize("name", mf.GRADED_ZIPS)
def test_compute_scene_metrics_is_the_benchmarks(tree, oracle_kernel, name):
    from zipfile import ZipFile
    with ZipFile(mf.write_zip(tree, name)) as zf:
        for scene in FIX["scene_order"]:
            res, failures = mfe.compute_scene_metrics(tree / "val", zf, scene)
            ref = FIX["zips"][name]["scenes"][scene]
            assert failures == ref["failures"]
            assert list(res) == list(ref["results"])
            for k in res:
                assert close(res[k], ref["results"][k]), (scene, k)


@pytest.mark.parametrize("name", mf.GRADED_ZIPS)
def test_cli_prints_the_benchmarks_json(tree, oracle_kernel, capsys, name):
    zp = mf.write_zip(tree, name)
    assert mfe.main(["--submission_path", str(zp), "--split", "val", "--dataset_path", str(tree)]) == 0
    ours = json.loads(capsys.readouterr().out)
    ref = FIX["zips"][name]["output"]
    assert list(ours) == list(ref)
    assert all(close(ours[k], ref[k]) for k in ref), {k: (ours[k], ref[k]) for k in ref}


def test_evaluate_submission_batches_as_one_call_per_image_size(tree, monkeypatch):
    calls = []

    def counting(*args):
        calls.append((len(args[0]), args[5], args[6]))
        return orc.frame_metrics(*args)
    monkeypatch.setattr(mfe, "frame_metrics", counting)
    out, curves = mfe.evaluate_submission(tree, mf.write_zip(tree, "near_perfect"), "val")
    assert sorted(calls) == [(5, 960, 540), (17, 540, 720)]
    assert close(out["AUC @ VCRE < 90px"], FIX["zips"]["near_perfect"]["output"]["AUC @ VCRE < 90px"])
    assert set(curves) == {"vcre_prec_values", "vcre_recall_values", "pose_prec_values", "pose_recall_values"}


def test_extra_scenes_and_missing_frames_are_logged(tree, oracle_kernel, caplog):
    with caplog.at_level(logging.WARNING, logger="mickey_b200.mapfree_eval"):
        mfe.evaluate_submission(tree, mf.write_zip(tree, "malformed_and_missing"), "val")
    text = caplog.text
    assert "estimates for 1 scenes outside the val set" in text
    failures = sum(v["failures"] for v in FIX["zips"]["malformed_and_missing"]["scenes"].values())
    assert failures == 19 and f"missing pose estimates for {failures} frames" in text
    assert "does not have estimates for scene s00003" in text


def test_no_valid_estimate_fails_with_the_benchmarks_message(tree, oracle_kernel, caplog, capsys):
    zp = mf.write_zip(tree, "no_valid_estimates")
    with pytest.raises(mfe.NoValidEstimates, match="Submission does not have any valid pose estimates"):
        mfe.evaluate_submission(tree, zp, "val")
    with caplog.at_level(logging.ERROR):
        assert mfe.main(["--submission_path", str(zp), "--split", "val", "--dataset_path", str(tree)]) == 1
    assert "Submission does not have any valid pose estimates" in caplog.text
    assert capsys.readouterr().out == FIX["zips"]["no_valid_estimates"]["stdout"] == ""


def test_a_negative_confidence_names_its_scene_and_frame(tree, oracle_kernel):
    with pytest.raises(ValueError, match="scene s00001 frame 10"):
        mfe.evaluate_submission(tree, mf.write_zip(tree, "negative_confidence"), "val")


def test_precision_recall_tie_rule_and_end_point():
    conf = [3.0, 1.0, 3.0, 0.0, 2.0, 0.0]
    tp = [True, False, False, True, True, False]
    prec, rec, auc = mfe.precision_recall(conf, tp, failures=2)
    # one point per distinct confidence (3, 2, 1, 0), cut at the first point of full recall, closed with (1, 0)
    assert rec.dtype == np.float32
    assert np.allclose(rec, [6 / 8, 4 / 8, 3 / 8, 2 / 8, 0]) and np.allclose(prec, [3 / 6, 2 / 4, 2 / 3, 1 / 2, 1])
    assert np.isclose(auc, 2 / 8 * 1 / 2 + 1 / 8 * 2 / 3 + 1 / 8 * 1 / 2 + 2 / 8 * 1 / 2)
