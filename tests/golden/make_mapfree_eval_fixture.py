"""Record the Map-free benchmark's grading (benchmark/mapfree.py of the unmodified reference, nianticlabs/mickey) on a small
val tree and a set of crafted submissions:

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_mapfree_eval_fixture.py

  reference_mapfree_eval.json
    "split", "scene_order"       the split and the order in which the benchmark walked the scene directories
    "scenes"                     scene -> {"intrinsics.txt": text, "poses.txt": text}: four scenes, one of them 960 x 540
    "gt_parsed"                  scene -> load_poses(poses.txt) as [frame, q (4), t (3)] rows in dict order (camera-to-world)
    "zips"                       name -> {"files": {member: text}, "parsed": {member: [frame, q, t, confidence] rows},
                                          "scenes": {scene: {"failures": n, "results": {metric: [values]}}},
                                          "stdout": what `python -m benchmark.mapfree` printed, "output": its JSON or null}

The crafted submissions (seeded, see crafted()) cover near-perfect poses, large errors, rotations near 180 degrees, estimates
that put grid points behind the camera, tied and zero confidences, non-unit quaternions, a missing frame, a missing
scene, an extra scene, a comment line, a wrong field count, NaN and infinite fields, a zero quaternion, a repeated frame,
and a submission with no valid estimate.  "negative_confidence" is recorded without a result: the benchmark's Inputs
assertion rejects it.  Only data is stored; transforms3d comes from compat/ when it is not installed.
"""
import contextlib
import io
import json
import os
import sys
import tempfile
import zipfile
from argparse import Namespace
from pathlib import Path

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF_ROOT = os.environ.get("MICKEY_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "reference_mapfree_eval.json")

# scene -> (seq1 frames in poses.txt, W, H, fx, fy, cx, cy): the intrinsics are not float32 values, so K's rounding shows
SCENES = {"s00000": (26, 540, 720, 590.137, 591.911, 269.23, 352.217),
          "s00001": (31, 540, 720, 602.5, 602.5, 271.731, 358.09),
          "s00002": (21, 960, 540, 745.003, 744.81, 481.377, 268.66),
          "s00003": (16, 540, 720, 588.8, 589.2, 268.1, 350.95)}


def axis_angle_q(axis, angle):
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * axis])


def qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 + y1 * w2 + z1 * x2 - x1 * z2, w1 * z2 + z1 * w2 + x1 * y2 - y1 * x2])


def gt_tree(rng):
    """scene -> ({file: text}, [(name, q, t)] of the seq1 frames)."""
    out = {}
    for scene, (n, W, H, fx, fy, cx, cy) in SCENES.items():
        names = ["seq0/frame_00000.jpg"] + [f"seq1/frame_{i:05d}.jpg" for i in range(n)]
        intr = "".join(f"{nm} {fx} {fy} {cx} {cy} {W} {H}\n" for nm in names)
        lines, frames = ["# frame qw qx qy qz tx ty tz (world to camera)"], []
        for i, nm in enumerate(names):
            if i == 0:
                q, t = np.array([1.0, 0, 0, 0]), np.zeros(3)
            else:
                q = axis_angle_q(rng.normal(size=3), np.deg2rad(rng.uniform(0, 25)))
                t = rng.uniform(-1.5, 1.5, size=3)
                q, t = np.round(q, 6), np.round(t, 6)
                frames.append((nm, q, t))
            lines.append(nm + " " + " ".join(f"{v:.6f}" for v in np.concatenate([q, t])))
        out[scene] = ({"intrinsics.txt": intr, "poses.txt": "\n".join(lines) + "\n"}, frames)
    return out


def line(name, q, t, conf, six=False):
    vals = list(q) + list(t)
    txt = " ".join(f"{v:.6f}" if six else repr(float(v)) for v in vals)
    return f"{name} {txt} {conf}"


def perturbed(rng, q, t, angle, dt):
    return qmul(q, axis_angle_q(rng.normal(size=3), angle)), t + rng.normal(size=3) * dt


def est_near_perfect(rng, q, t, i):
    q, t = perturbed(rng, q, t, 10 ** rng.uniform(-3, -2), 10 ** rng.uniform(-3, -2))
    return q, t, repr(float(rng.uniform(100, 1000)))


def est_large(rng, q, t, i):
    return axis_angle_q(rng.normal(size=3), rng.uniform(0, np.pi)), rng.uniform(-5, 5, size=3), str(int(rng.integers(0, 500)))


def est_near_180(rng, q, t, i):
    q = qmul(q, axis_angle_q(rng.normal(size=3), np.pi - 10 ** rng.uniform(-6, -2)))
    return q, t + rng.normal(size=3) * 0.05, repr(float(rng.uniform(0, 50)))


def est_behind(rng, q, t, i):
    # turn the estimate 60-150 degrees about its y axis and move it 1.5-3 m along z: part of the grid lands behind it
    q = qmul(axis_angle_q([0, 1, 0], np.deg2rad(rng.uniform(60, 150)) * rng.choice([-1, 1])), q)
    return q, t + np.array([0, 0, -rng.uniform(1.5, 3.0)]), repr(float(rng.uniform(1, 9)))


def est_ties(rng, q, t, i):
    q, t = perturbed(rng, q, t, np.deg2rad(rng.uniform(0, 10)), rng.uniform(0, 0.3))
    return q, t, str(rng.choice(["0", "0", "0.0", "5", "5.0", "5", "17", "17", "300"]))


def est_nonunit(rng, q, t, i):
    q, t = perturbed(rng, q, t, np.deg2rad(rng.uniform(0, 8)), rng.uniform(0, 0.4))
    return q * rng.uniform(0.3, 3.0), t, repr(float(rng.uniform(0, 100)))


def scene_file(rng, frames, est, six=False):
    return "\n".join(line(nm, *est(rng, q, t, i), six=six) for i, (nm, q, t) in enumerate(frames))


def crafted(rng, gt):
    zips = {}
    for name, est in (("near_perfect", est_near_perfect), ("large_errors", est_large), ("near_180", est_near_180),
                      ("behind_camera", est_behind), ("confidence_ties", est_ties), ("nonunit_quaternions", est_nonunit)):
        zips[name] = {f"pose_{s}.txt": scene_file(rng, frames, est, six=name == "confidence_ties")
                      for s, (_, frames) in gt.items()}
    # malformed lines, a missing frame, a missing scene (s00003) and an extra one
    f0 = gt["s00000"][1]
    good = [line(nm, *est_ties(rng, q, t, i)) for i, (nm, q, t) in enumerate(f0)]
    bad = ["#" + f0[0][0] + " 1 0 0 0 0 0 0 3",                             # comment (9 fields)
           f0[5][0] + " 1 0 0 0 0 0 0",                                    # 8 fields: too few
           f0[5][0] + " 1 0 0 0 0 0 0 3 4",                                # 10 fields: too many
           f0[10][0] + " nan 0 0 0 0 0 0 3",                               # NaN (frame 10 keeps its good line)
           f0[10][0] + " 1 0 0 0 inf 0 0 3",                               # infinite
           f0[15][0] + " 0 0 0 0 0.1 0.2 0.3 3",                           # zero quaternion: frame 15 becomes a failure
           f0[20][0] + " 1 0 0 0 0 0 0 2"]                                 # replaced by its second line below
    s0 = [bad[0]] + good[:5] + [bad[1], bad[2], bad[3], bad[4]] + good[10:15] + [bad[5]] + good[16:20] + [bad[6]] + \
         good[20:]
    s0 = [ln for ln in s0 if not ln.startswith(f0[25][0])]                   # frame 25: no line at all
    zips["malformed_and_missing"] = {
        "pose_s00000.txt": "\n".join(s0),
        "pose_s00001.txt": scene_file(rng, gt["s00001"][1], est_ties),
        "pose_s00002.txt": scene_file(rng, gt["s00002"][1], est_near_perfect),
        "pose_s09999.txt": scene_file(rng, gt["s00001"][1], est_large)}
    zips["no_valid_estimates"] = {"pose_s09999.txt": scene_file(rng, gt["s00001"][1], est_large)}
    neg = scene_file(rng, gt["s00001"][1], est_ties).split("\n")
    neg[10] = neg[10].rsplit(" ", 1)[0] + " -1.5"                            # frame 10 (graded) with confidence -1.5
    zips["negative_confidence"] = {f"pose_{s}.txt": scene_file(rng, frames, est_ties) for s, (_, frames) in gt.items()}
    zips["negative_confidence"]["pose_s00001.txt"] = "\n".join(neg)
    return zips


def rows(poses, conf):
    return [[int(k), [float(x) for x in q], [float(x) for x in t]] + ([float(c)] if conf else [])
            for k, (q, t, c) in poses.items()]


def record():
    compat = [os.path.join(ROOT, "compat")] if __import__("importlib").util.find_spec("transforms3d") is None else []
    sys.path[:0] = [REF_ROOT] + compat + [ROOT]
    from benchmark import mapfree as bm
    from benchmark.utils import load_poses

    rng = np.random.default_rng(20261017)
    gt = gt_tree(rng)
    zips = crafted(rng, gt)
    out = {"split": "val", "scenes": {s: files for s, (files, _) in gt.items()}, "gt_parsed": {}, "zips": {}}
    with tempfile.TemporaryDirectory() as tmp:
        split = Path(tmp) / "val"
        for s, (files, _) in gt.items():
            (split / s).mkdir(parents=True)
            for fn, text in files.items():
                (split / s / fn).write_text(text)
            with (split / s / "poses.txt").open() as f:
                out["gt_parsed"][s] = rows(load_poses(f, load_confidence=False), False)
        out["scene_order"] = [f.name for f in split.iterdir() if f.is_dir()]
        for name, files in zips.items():
            zp = Path(tmp) / f"{name}.zip"
            with zipfile.ZipFile(zp, "w") as zf:
                for fn, text in files.items():
                    zf.writestr(fn, text.encode("utf-8"))
            rec = {"files": files, "parsed": {}}
            for fn, text in files.items():
                f = io.StringIO(text)
                f.name = fn
                rec["parsed"][fn] = rows(load_poses(f, load_confidence=True), True)
            if name != "negative_confidence":
                with zipfile.ZipFile(zp) as zf:
                    rec["scenes"] = {}
                    for s in out["scene_order"]:
                        res, failures = bm.compute_scene_metrics(split, zf, s)
                        rec["scenes"][s] = {"failures": int(failures),
                                            "results": {k: [float(v) for v in vs] for k, vs in res.items()}}
                buf = io.StringIO()
                with contextlib.redirect_stdout(buf):
                    bm.main(Namespace(dataset_path=Path(tmp), split="val", submission_path=zp))
                rec["stdout"] = buf.getvalue()
                rec["output"] = json.loads(buf.getvalue()) if buf.getvalue().strip() else None
            out["zips"][name] = rec
    with open(OUT, "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print("wrote", OUT, {k: (v.get("output") or {}).get("AUC @ VCRE < 90px") for k, v in out["zips"].items()})


if __name__ == "__main__":
    record()
