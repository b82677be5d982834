"""mk_mapfree_frame_metrics on the GPU: per-frame errors against the fp64 oracle on every fixture frame and on 100 000
seeded random frames, the bits of a frame alone, in a batch and across runs, whole submissions against the benchmark's
recorded JSON, and tools/run_submission.py --evaluate on a synthetic val tree.

Tolerances against the oracle:
  trans_err, reproj_err  1e-12 relative.  Two exceptions are counted and reported, not failed: a frame with a grid point
                         whose depth lies within 1e-12 of zero (a last-bit difference there can move the clipped
                         projection from one image border to the other), and a difference within 64 ulp of the operands
                         the error is a difference of (the camera centres for trans_err, the pixel coordinates, at most
                         max(W, H), for reproj_err): a near-perfect estimate's error cannot be more accurate than its
                         operands.  The fixture frames need neither.
  rot_err                1e-9 degrees where |vec| = sin(rot_err / 2) < 1 - 1e-6.  Nearer 180 degrees asin is
                         ill-conditioned (d asin(s)/ds = 1/sqrt(1 - s^2)); there the bound is the change of asin under a
                         perturbation of s by DELTA = 1e-14 (some ten times the rounding of |vec|):
                         114.59 * (asin(min(s + DELTA, 1)) - asin(max(s - DELTA, 0))) + 1e-9, and a NaN (s rounded above
                         1) is accepted on one side only where 1 - s < DELTA.
"""
import json
import logging
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "compat")) if __import__("importlib").util.find_spec("transforms3d") is None else None

from mickey_b200 import mapfree_eval as mfe  # noqa: E402
from oracle import mapfree_eval_oracle as orc  # noqa: E402
from tests import mapfree_fixture as mf  # noqa: E402

pytestmark = pytest.mark.gpu
DELTA = 1e-14
EPS = np.finfo(np.float64).eps
DEG = 114.59155902616465


def kernel(q_est, t_est, q_gt, t_gt, K, W, H):
    return mfe.frame_metrics(q_est, t_est, q_gt, t_gt, K, W, H)


def rot_bound(rot_ref):
    s = np.sin(rot_ref / DEG)
    near = s >= 1 - 1e-6
    wide = DEG * (np.arcsin(np.minimum(s + DELTA, 1)) - np.arcsin(np.maximum(s - DELTA, 0))) + 1e-9
    return np.where(near, wide, 1e-9), s


def residual_depths(q_est, t_est, q_gt, t_gt, K):
    """The depth row of K (M X) for every frame and grid point, [P, 196]."""
    out = np.empty((len(q_est), 196))
    for i in range(len(q_est)):
        qe, ce = orc.world2cam_to_cam2world(q_est[i], t_est[i])
        qg, cg = orc.world2cam_to_cam2world(q_gt[i], t_gt[i])
        E, G = np.eye(4), np.eye(4)
        E[:3, :3], E[:3, 3], G[:3, :3], G[:3, 3] = orc.quat2mat(qe), ce, orc.quat2mat(qg), cg
        out[i] = K[i][2] @ (np.linalg.inv(E) @ G @ orc._EYE.T)[:3]
    return out


def compare(got, ref, q_est, t_est, q_gt, t_gt, K, W, H):
    """Assert the module docstring's tolerances; return the counts of frames that used an exception."""
    assert got.shape == ref.shape
    rel = np.abs(got - ref) <= 1e-12 * np.abs(ref)
    centres = np.array([np.linalg.norm(orc.world2cam_to_cam2world(q, t)[1]) for q, t in zip(q_est, t_est)]) + \
        np.array([np.linalg.norm(orc.world2cam_to_cam2world(q, t)[1]) for q, t in zip(q_gt, t_gt)])
    floor = {0: 64 * EPS * centres, 2: 64 * EPS * max(W, H) * np.ones(len(ref))}
    near_zero = np.zeros(len(ref), dtype=bool)
    if not rel[:, [0, 2]].all():
        near_zero = (np.abs(residual_depths(q_est, t_est, q_gt, t_gt, K)) < 1e-12).any(1)
    counts = {"depth_near_zero": int(near_zero.sum())}
    for c in (0, 2):
        ok_floor = np.abs(got[:, c] - ref[:, c]) <= floor[c]
        bad = ~(rel[:, c] | ok_floor | (near_zero if c == 2 else False))
        assert not bad.any(), (c, np.flatnonzero(bad)[:5], got[bad][:5], ref[bad][:5])
        counts[f"floor_{c}"] = int((~rel[:, c] & ok_floor).sum())
    bound, s = rot_bound(ref[:, 1])
    nan_got, nan_ref = np.isnan(got[:, 1]), np.isnan(ref[:, 1])
    both = ~nan_got & ~nan_ref
    assert (np.abs(got[both, 1] - ref[both, 1]) <= bound[both]).all(), \
        np.max(np.abs(got[both, 1] - ref[both, 1]) / bound[both])
    assert not (nan_got & ~nan_ref & (1 - s >= DELTA)).any()
    counts["near_180"] = int((s >= 1 - 1e-6).sum())
    return counts


# ---- the fixture's frames ---------------------------------------------------------------------------------------------------
def fixture_frames(tmp_path):
    """Every graded frame of every fixture zip, grouped by image size: {(W, H): (q_est, t_est, q_gt, t_gt, K)}."""
    root = mf.write_tree(tmp_path)
    groups = {}
    for z in mf.GRADED_ZIPS:
        for _, fr in mf.graded_frames(root, z):
            g = groups.setdefault((int(fr["W"]), int(fr["H"])), [[] for _ in range(5)])
            for lst, k in zip(g, ("q_est", "t_est", "q_gt", "t_gt", "K")):
                lst.append(fr[k])
    return {wh: [np.concatenate(v) for v in g] for wh, g in groups.items()}


def test_fixture_frames_against_the_oracle(tmp_path):
    total = 0
    for (W, H), args in fixture_frames(tmp_path).items():
        got, ref = kernel(*args, W, H), orc.frame_metrics(*args, W, H)
        counts = compare(got, ref, *args, W, H)
        print(f"{W}x{H}: {len(ref)} fixture frames, exceptions used: {counts}")
        assert counts["depth_near_zero"] == 0 and counts["floor_0"] == 0 and counts["floor_2"] == 0
        total += len(ref)
    assert total == sum(len(s["results"].get("trans_err", [])) for z in mf.GRADED_ZIPS
                        for s in mf.FIX["zips"][z]["scenes"].values())


# ---- seeded random frames -------------------------------------------------------------------------------------------------
def random_frames(n, seed=0):
    """World-to-camera estimates and ground truths: unit and non-unit quaternions, relative rotations from 1e-3 rad to
    180 degrees, centre offsets from 1 cm to 5 m, float32 intrinsics."""
    rng = np.random.default_rng(seed)

    def unit(size):
        v = rng.normal(size=(size, 4))
        return v / np.linalg.norm(v, axis=1, keepdims=True)
    q_gt = unit(n) * np.where(rng.random((n, 1)) < 0.3, rng.uniform(0.5, 2.0, (n, 1)), 1.0)
    axis = rng.normal(size=(n, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    ang = np.where(rng.random(n) < 0.5, 10 ** rng.uniform(-3, -0.5, n), rng.uniform(0, np.pi, n))
    dq = np.concatenate([np.cos(ang / 2)[:, None], np.sin(ang / 2)[:, None] * axis], 1)
    q_est = np.stack([orc.qmult(a, b) for a, b in zip(q_gt, dq)]) * np.where(rng.random((n, 1)) < 0.3,
                                                                              rng.uniform(0.5, 2.0, (n, 1)), 1.0)
    t_gt = rng.uniform(-3, 3, (n, 3))
    t_est = t_gt + rng.normal(size=(n, 3)) * 10 ** rng.uniform(-2, 0.7, (n, 1))
    f = rng.uniform(300, 1000, n)
    K = np.zeros((n, 3, 3))
    K[:, 0, 0], K[:, 1, 1] = f, f * rng.uniform(0.98, 1.02, n)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = 270 + rng.uniform(-20, 20, n), 360 + rng.uniform(-20, 20, n), 1
    return q_est, t_est, q_gt, t_gt, K.astype(np.float32).astype(np.float64)


def test_100k_random_frames_against_the_oracle():
    args = random_frames(100_000)
    got, ref = kernel(*args, 540, 720), orc.frame_metrics(*args, 540, 720)
    counts = compare(got, ref, *args, 540, 720)
    print("100000 random frames (12500 blocks of 8 frames), exceptions used:", counts)


def test_a_frames_bits_do_not_depend_on_the_batch_or_the_run():
    args = random_frames(4096, seed=1)
    once, twice = kernel(*args, 540, 720), kernel(*args, 540, 720)
    assert once.tobytes() == twice.tobytes()
    perm = np.random.default_rng(2).permutation(4096)
    shuffled = kernel(*(a[perm] for a in args), 540, 720)
    assert shuffled.tobytes() == once[perm].tobytes()
    for i in (0, 1, 7, 8, 9, 31, 4095):
        alone = kernel(*(a[i:i + 1] for a in args), 540, 720)
        assert alone.tobytes() == once[i:i + 1].tobytes()
    tail = kernel(*(a[4000:] for a in args), 540, 720)
    assert tail.tobytes() == once[4000:].tobytes()


def test_the_kernel_runs_on_the_callers_stream():
    args = [torch.from_numpy(a).cuda() for a in random_frames(1000, seed=3)]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out = mfe.frame_metrics_dev(*args, 540, 720)
    s.synchronize()
    assert torch.equal(out.cpu(), torch.from_numpy(kernel(*(a.cpu().numpy() for a in args), 540, 720)))


# ---- whole submissions --------------------------------------------------------------------------------------------------------
def assert_same_metrics(ours, ref, rot_values):
    """Every number within 1e-12 relative; the average median rotation error within 1e-12 relative plus the largest
    per-frame rotation bound (a median of values that are each within their bound is within the largest bound)."""
    assert list(ours) == list(ref)
    extra = rot_bound(np.asarray(rot_values))[0].max() if len(rot_values) else 0.0
    for k in ref:
        tol = 1e-12 * abs(ref[k]) + (extra if k == "Average Median Rotation Error" else 0.0)
        assert abs(ours[k] - ref[k]) <= tol, (k, ours[k], ref[k])


@pytest.mark.parametrize("name", mf.GRADED_ZIPS)
def test_evaluate_submission_prints_the_fixtures_json(tmp_path, capsys, name):
    root = mf.write_tree(tmp_path)
    zp = mf.write_zip(root, name)
    assert mfe.main(["--submission_path", str(zp), "--split", "val", "--dataset_path", str(root)]) == 0
    ours = json.loads(capsys.readouterr().out)
    rot = [v for s in mf.FIX["zips"][name]["scenes"].values() for v in s["results"].get("rot_err", [])]
    assert_same_metrics(ours, mf.FIX["zips"][name]["output"], rot)


def test_run_submission_evaluate_on_a_synthetic_val_tree(tmp_path, monkeypatch):
    from mickey_b200.config import CfgNode, mickey_cfg
    from tools.make_synthetic_mapfree import make_tree
    cfg = mickey_cfg("vits", 2, 8)
    (tmp_path / "model.yaml").write_text(CfgNode({k: cfg[k] for k in ("MODEL", "MICKEY", "FEATURE_MATCHER", "PROCRUSTES")}).dump())
    make_tree(str(tmp_path / "data"), "val", scenes=2, queries=20, seed=5)

    def run(out, *extra):
        cmd = [sys.executable, os.path.join(ROOT, "tools", "run_submission.py"), "--variant", "vits", "--config",
               str(tmp_path / "model.yaml"), "--checkpoint", "synthetic", "--data_root", str(tmp_path / "data"),
               "--split", "val", "--workers", "0", "--seed", "11", "-o", str(tmp_path / out), *extra]
        r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT),
                           timeout=900)
        assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
        return json.loads(r.stdout.strip().splitlines()[-1])

    plain, graded = run("plain"), run("graded", "--evaluate")
    # without the flag: the summary's keys and values are what they were; only the clocks differ
    assert list(plain) == [k for k in graded if k != "mapfree_metrics"]
    differ = {"wall_s", "pairs_per_s", "zip"}          # the clocks, and the output directory the two runs were given
    assert {k: v for k, v in plain.items() if k not in differ} == {k: v for k, v in graded.items()
                                                                   if k not in differ | {"mapfree_metrics"}}
    zp = tmp_path / "graded" / "submission.zip"
    from zipfile import ZipFile

    def members(path):
        with ZipFile(path) as z:
            return {n: z.read(n) for n in z.namelist()}
    assert members(tmp_path / "plain" / "submission.zip") == members(zp)      # (the headers hold the write time)
    metrics = graded["mapfree_metrics"]
    assert plain["pairs"] == 8 and metrics["Estimates for % of frames"] > 0
    # the CLI on the same zip: the same kernel, the same bits
    cli = subprocess.run([sys.executable, "-m", "mickey_b200.mapfree_eval", "--submission_path", str(zp), "--split",
                          "val", "--dataset_path", str(tmp_path / "data")], capture_output=True, text=True, cwd=ROOT,
                         timeout=600)
    assert cli.returncode == 0, cli.stderr[-3000:]
    assert json.loads(cli.stdout) == metrics
    # and the oracle in the kernel's place
    monkeypatch.setattr(mfe, "frame_metrics", orc.frame_metrics)
    logging.disable(logging.WARNING)
    try:
        ours, _ = mfe.evaluate_submission(tmp_path / "data", zp, "val")
    finally:
        logging.disable(logging.NOTSET)
    split = tmp_path / "data" / "val"
    with ZipFile(zp) as zf:
        rot = [v for s in ("s00000", "s00001") for v in mfe.compute_scene_metrics(split, zf, s)[0].get("rot_err", [])]
    assert_same_metrics(metrics, ours, rot)
