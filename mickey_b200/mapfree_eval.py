"""Grade a Map-free submission as the benchmark does (benchmark/mapfree.py with benchmark/metrics.py, reprojection.py and
utils.py), with the per-frame errors computed by one CUDA kernel (mk_mapfree_frame_metrics) over every graded frame:

    python -m mickey_b200.mapfree_eval --submission_path results/submission.zip --split val --dataset_path data/

prints the JSON that `python -m benchmark.mapfree` prints: precision and AUC at VCRE < 90 px and at pose error
< (25 cm, 5 deg), the average per-scene medians of the three errors and the share of frames with an estimate.

The host logic is the benchmark's, rules and quirks included: the pose-file parser's skipping rules, the subsampling of
the ground truth by enumeration order, failures counted before subsampling for a scene the zip lacks, medians over the
scenes that have results only, and the precision/recall curve's tie rule, float32 recall and end point.  Only the
per-frame errors leave the host; the aggregation is a few thousand values per split and stays numpy fp64.
"""
from __future__ import annotations

import argparse
import json
import logging
import os
import sys
from collections import defaultdict
from io import TextIOWrapper
from pathlib import Path
from zipfile import ZipFile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# thresholds of benchmark/config.py
T_THRESHOLD = 0.25          # metres
R_THRESHOLD = 5             # degrees
VCRE_THRESHOLD = 90         # pixels
SUBSAMPLE = 5               # the val / test ground truth is graded on every 5th frame
METRICS = ("trans_err", "rot_err", "reproj_err", "confidence")      # MetricManager's order

log = logging.getLogger("mickey_b200.mapfree_eval")


# ---- the benchmark's file rules ----------------------------------------------------------------------------------------
def load_poses(file, load_confidence: bool = False) -> dict:
    """Pose lines `<name> qw qx qy qz tx ty tz [confidence]` -> {frame number: (q [4], t [3], confidence or None)}, kept
    world-to-camera (mk_mapfree_frame_metrics converts them).  As in benchmark/utils.py::load_poses, a line is skipped
    when it has the wrong number of fields, when its name holds a '#' (a comment), when the frame number name[-9:-4] is
    not an integer, when a value is NaN or infinite, or when the quaternion's norm is close to zero; a later line for the
    same frame replaces the earlier one but keeps its place in the order."""
    expected = 9 if load_confidence else 8
    where = getattr(file, "name", "<pose file>")
    poses = {}
    for line_number, line in enumerate(file.readlines()):
        parts = line.strip().split(" ")
        if len(parts) != expected:
            log.warning("%s line %d: %d fields, expected %d; line ignored", where, line_number, len(parts), expected)
            continue
        name = parts[0]
        if "#" in name:
            log.info("%s line %d: comment ignored", where, line_number)
            continue
        try:
            frame = int(name[-9:-4])
        except ValueError:
            log.warning("%s line %d: no frame number in %r; line ignored", where, line_number, name)
            continue
        try:
            values = [float(v) for v in parts[1:]]
        except ValueError:
            log.warning("%s line %d: unparsable pose; line ignored", where, line_number)
            continue
        if not all(np.isfinite(values)):
            log.warning("%s line %d: NaN or infinite value; line ignored", where, line_number)
            continue
        q, t = np.array(values[:4], dtype=np.float64), np.array(values[4:7], dtype=np.float64)
        if np.isclose(np.linalg.norm(q), 0):
            log.warning("%s line %d: quaternion of zero norm; line ignored", where, line_number)
            continue
        poses[frame] = (q, t, values[7] if load_confidence else None)
    return poses


def subsample_poses(poses: dict, subsample: int = 1) -> dict:
    """Every `subsample`-th entry in the dict's order."""
    return {k: v for i, (k, v) in enumerate(poses.items()) if i % subsample == 0}


def load_K(file_path: Path):
    """intrinsics.txt -> ({frame number: K [3, 3] float32}, W, H), with K rounded to float32 and W, H taken from the last
    line, as benchmark/utils.py::load_K does.  The rows are those of the dataset's own parser."""
    from lib.datasets.mapfree import _rows
    K, W, H = {}, None, None
    for name, (fx, fy, cx, cy, W, H) in _rows(Path(file_path)):
        K[int(name[-9:-4])] = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float32)
    return K, W, H


def count_unexpected_scenes(scenes, submission_zip: ZipFile) -> int:
    in_zip = {n[5:-4] for n in submission_zip.namelist() if n.startswith("pose_")}
    return len(in_zip - set(scenes))


# ---- per-frame errors on the GPU -----------------------------------------------------------------------------------------
_grids = {}


def _grid(dev):
    if dev not in _grids:
        from mickey_b200.loss import vcre_grid
        _grids[dev] = vcre_grid(dev).contiguous()
    return _grids[dev]


def frame_metrics_dev(q_est, t_est, q_gt, t_gt, K, W: int, H: int, out=None):
    """mk_mapfree_frame_metrics on CUDA fp64 tensors q_est [P, 4], t_est [P, 3], q_gt [P, 4], t_gt [P, 3], K [P, 3, 3]
    (world-to-camera poses), clipped to a W x H image -> fp64 [P, 3] = trans_err, rot_err, reproj_err, enqueued on the
    current stream."""
    import torch
    from mickey_b200 import _lib
    P = q_est.shape[0]
    shapes = {"q_est": (q_est, (P, 4)), "t_est": (t_est, (P, 3)), "q_gt": (q_gt, (P, 4)), "t_gt": (t_gt, (P, 3)),
              "K": (K, (P, 3, 3))}
    dev = q_est.device
    for name, (t, shape) in shapes.items():
        if tuple(t.shape) != shape or t.dtype != torch.float64 or t.device != dev or not t.is_contiguous():
            raise ValueError(f"{name}: need a contiguous fp64 {shape} tensor on {dev}, got {t.dtype} "
                             f"{tuple(t.shape)} on {t.device}")
    if dev.type != "cuda":
        raise ValueError(f"mk_mapfree_frame_metrics runs on a CUDA device, got {dev}")
    if out is None:
        out = torch.empty(P, 3, dtype=torch.float64, device=dev)
    lib = _lib.load()
    _lib.check(lib.mk_mapfree_frame_metrics(_lib.ptr(q_est), _lib.ptr(t_est), _lib.ptr(q_gt), _lib.ptr(t_gt),
                                            _lib.ptr(K), _lib.ptr(_grid(dev)), P, int(W), int(H), _lib.ptr(out),
                                            _lib.stream(dev)), "mk_mapfree_frame_metrics")
    return out


def frame_metrics(q_est, t_est, q_gt, t_gt, K, W, H) -> np.ndarray:
    """Numpy in, numpy out: the frames' errors [P, 3] computed on the current CUDA device."""
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    args = [torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev) for a in (q_est, t_est, q_gt, t_gt, K)]
    return frame_metrics_dev(*args, W, H).cpu().numpy()


# ---- grading ----------------------------------------------------------------------------------------------------------------
def _scene_frames(split_path: Path, submission_zip: ZipFile, scene: str):
    """The graded frames of one scene -> (frames or None when the zip has no file for the scene, failures).  frames holds
    stacked q_est, t_est, q_gt, t_gt, K, confidence, W and H."""
    K, W, H = load_K(split_path / scene / "intrinsics.txt")
    with (split_path / scene / "poses.txt").open("r", encoding="utf-8") as f:
        gt = load_poses(f, load_confidence=False)
    try:
        with submission_zip.open(f"pose_{scene}.txt") as f:
            est = load_poses(TextIOWrapper(f, encoding="utf-8"), load_confidence=True)
    except KeyError:
        log.warning("Submission does not have estimates for scene %s.", scene)
        return None, len(gt)                     # counted before subsampling, as the benchmark does
    rows, failures = [], 0
    for frame, (q, t, _) in subsample_poses(gt, SUBSAMPLE).items():
        if frame not in est:
            failures += 1
            continue
        qe, te, conf = est[frame]
        if not conf >= 0:
            raise ValueError(f"scene {scene} frame {frame}: confidence {conf} is negative; the benchmark requires >= 0")
        rows.append((qe, te, q, t, K[frame], conf))
    cols = list(zip(*rows)) if rows else [()] * 6
    shapes = ((4,), (3,), (4,), (3,), (3, 3))
    frames = {k: np.array(c, dtype=np.float64).reshape((-1,) + s)
              for k, c, s in zip(("q_est", "t_est", "q_gt", "t_gt", "K"), cols, shapes)}
    frames["confidence"] = list(cols[5])
    frames["W"], frames["H"] = W, H
    return frames, failures


def _image_size(frames):
    W, H = frames["W"], frames["H"]
    if W != int(W) or H != int(H):
        raise ValueError(f"image size {W} x {H} is not integral")
    return int(W), int(H)


def _grade(frames_list):
    """Per-frame errors of every scene's frames, one kernel launch per distinct image size."""
    groups = defaultdict(list)
    for i, fr in enumerate(frames_list):
        if len(fr["confidence"]):
            groups[_image_size(fr)].append(i)
    errs = [np.zeros((0, 3)) for _ in frames_list]
    for (W, H), idx in groups.items():
        cat = [np.concatenate([frames_list[i][k] for i in idx]) for k in ("q_est", "t_est", "q_gt", "t_gt", "K")]
        e = frame_metrics(*cat, W, H)
        ends = np.cumsum([len(frames_list[i]["confidence"]) for i in idx])
        for i, part in zip(idx, np.split(e, ends[:-1])):
            errs[i] = part
    return errs


def _results(frames, err):
    """MetricManager's per-scene dict: metric -> one value per graded frame."""
    results = defaultdict(list)
    for row, conf in zip(err, frames["confidence"]):
        for name, v in zip(METRICS, (row[0], row[1], row[2], conf)):
            results[name].append(v)
    return results


def compute_scene_metrics(dataset_path: Path, submission_zip: ZipFile, scene: str):
    """One scene of a split directory -> (results, failures): benchmark/mapfree.py::compute_scene_metrics."""
    frames, failures = _scene_frames(Path(dataset_path), submission_zip, scene)
    if frames is None:
        return dict(), failures
    return _results(frames, _grade([frames])[0]), failures


def precision_recall(inliers, tp, failures):
    """Precision / recall of the frames ranked by confidence, descending, one point per distinct confidence (the last
    frame of each tied run), recall over graded frames plus failures; the curve is reversed, cut at the first point of
    full recall and closed with (precision 1, recall 0).  Returns (precision, recall, AUC)."""
    if len(inliers) != len(tp):
        raise ValueError("precision_recall: unequal lengths")
    conf = np.array(inliers)
    order = np.argsort(conf)[::-1]
    conf = conf[order]
    hits = np.array(tp).reshape(-1)[order]
    run_ends = np.r_[np.where(np.diff(conf))[0], conf.size - 1]
    n = conf.shape[0]
    ranks = np.arange(n, dtype=np.float32) + 1
    prec = np.cumsum(hits)[run_ends] / ranks[run_ends]
    rec = ranks[run_ends] / (float(n) + float(failures))
    first_full = rec.searchsorted(rec[-1])
    prec = np.r_[prec[first_full::-1], 1]
    rec = np.r_[rec[first_full::-1], 0]
    return prec, rec, np.abs(np.sum(np.diff(rec) * prec[:-1]))


def aggregate_results(all_results: dict, all_failures: int):
    """{scene: results} and the failure count -> (output metrics, curves): benchmark/mapfree.py::aggregate_results."""
    medians, values = defaultdict(list), defaultdict(list)
    for scene_results in all_results.values():
        for metric, v in scene_results.items():
            medians[metric].append(np.median(v))
            values[metric].extend(v)
    values = {k: np.array(v) for k, v in values.items()}
    avg_median = {k: np.mean(v) for k, v in medians.items()}
    pose_ok = (values["trans_err"] < T_THRESHOLD) * (values["rot_err"] < R_THRESHOLD)
    vcre_ok = values["reproj_err"] < VCRE_THRESHOLD
    graded = len(values["trans_err"])
    total = graded + all_failures
    pose_prec, pose_rec, pose_auc = precision_recall(values["confidence"], pose_ok, all_failures)
    vcre_prec, vcre_rec, vcre_auc = precision_recall(values["confidence"], vcre_ok, all_failures)
    curves = {"vcre_prec_values": vcre_prec, "vcre_recall_values": vcre_rec,
              "pose_prec_values": pose_prec, "pose_recall_values": pose_rec}
    pose = f"({T_THRESHOLD * 100}cm, {R_THRESHOLD}deg)"
    out = {"Average Median Translation Error": avg_median["trans_err"],
           "Average Median Rotation Error": avg_median["rot_err"],
           "Average Median Reprojection Error": avg_median["reproj_err"],
           f"Precision @ Pose Error < {pose}": np.sum(pose_ok) / total,
           f"AUC @ Pose Error < {pose}": pose_auc,
           f"Precision @ VCRE < {VCRE_THRESHOLD}px": np.sum(vcre_ok) / total,
           f"AUC @ VCRE < {VCRE_THRESHOLD}px": vcre_auc,
           "Estimates for % of frames": graded / total}
    return out, curves


class NoValidEstimates(ValueError):
    pass


def evaluate_submission(dataset_path, submission_zip, split: str):
    """Grade `submission_zip` (a path or an open ZipFile) against <dataset_path>/<split>/ -> (output metrics, curves),
    the benchmark's numbers under its key strings.  Raises NoValidEstimates when no scene has a graded frame."""
    split_path = Path(dataset_path) / split
    scenes = tuple(f.name for f in split_path.iterdir() if f.is_dir())
    zf = submission_zip if isinstance(submission_zip, ZipFile) else ZipFile(submission_zip, "r")
    try:
        collected, all_failures = {}, 0
        for scene in scenes:
            collected[scene], failures = _scene_frames(split_path, zf, scene)
            all_failures += failures
        present = [s for s in scenes if collected[s] is not None]
        errs = _grade([collected[s] for s in present])
        all_results = {s: dict() for s in scenes}
        all_results.update({s: _results(collected[s], e) for s, e in zip(present, errs)})
        if all_failures > 0:
            log.warning("Submission is missing pose estimates for %d frames", all_failures)
        unexpected = count_unexpected_scenes(scenes, zf)
        if unexpected > 0:
            log.warning("Submission contains estimates for %d scenes outside the %s set", unexpected, split)
    finally:
        if zf is not submission_zip:
            zf.close()
    if all(len(r) == 0 for r in all_results.values()):
        raise NoValidEstimates("Submission does not have any valid pose estimates")
    return aggregate_results(all_results, all_failures)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser("mapfree_eval", description="Evaluate submissions for the MapFree dataset benchmark")
    ap.add_argument("--submission_path", type=Path, default="", help="Path to the submission ZIP file")
    ap.add_argument("--split", choices=("val", "test"), default="test",
                    help="Dataset split to use for evaluation. Default: test")
    ap.add_argument("--log", choices=("warning", "info", "error"), default="warning",
                    help="Logging level. Default: warning")
    ap.add_argument("--dataset_path", type=Path, default=None,
                    help="Path to the dataset folder (default: DATA_ROOT of config/datasets/mapfree.yaml)")
    args = ap.parse_args(argv)
    logging.basicConfig(level=args.log.upper())
    if args.dataset_path is None:
        from config.default import cfg
        cfg.merge_from_file(os.path.join(ROOT, "config", "datasets", "mapfree.yaml"))
        args.dataset_path = Path(cfg.DATASET.DATA_ROOT)
    if not args.submission_path.is_file():
        log.error("Could not find ZIP file in path %s", args.submission_path)
        return 1
    try:
        metrics, _ = evaluate_submission(args.dataset_path, args.submission_path, args.split)
    except NoValidEstimates as e:
        log.error("%s", e)
        return 1
    print(json.dumps(metrics, indent=2))
    return 0


if __name__ == "__main__":
    sys.path[:0] = [ROOT] + ([os.path.join(ROOT, "compat")]
                             if __import__("importlib").util.find_spec("transforms3d") is None else [])
    sys.exit(main())
