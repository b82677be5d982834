"""Time the grading of a val-sized Map-free submission (65 scenes x 115 graded frames by default) on the GPU:

    python tools/mapfree_eval_bench.py [--scenes 65 --graded 115 --reps 200]

The tree (poses.txt and intrinsics.txt only) and a submission with seeded random estimates are written to a temporary
directory.  Prints one JSON line: mk_mapfree_frame_metrics's time for all graded frames in one launch (CUDA events, median
over --reps launches), the wall time of evaluate_submission and of the CLI process on the zip, the oracle's host time for
the same frames as context, the device name and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zipfile
from pathlib import Path

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT] + ([os.path.join(ROOT, "compat")]
                         if __import__("importlib").util.find_spec("transforms3d") is None else [])


def write_split(root: Path, scenes: int, graded: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    frames = graded * 5
    for s in range(scenes):
        d = root / "val" / f"s{s:05d}"
        d.mkdir(parents=True)
        names = ["seq0/frame_00000.jpg"] + [f"seq1/frame_{i:05d}.jpg" for i in range(frames)]
        (d / "intrinsics.txt").write_text("".join(f"{n} 590.0 590.0 269.2 352.2 540 720\n" for n in names))
        q = rng.normal(size=(len(names), 4))
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        t = rng.uniform(-1.5, 1.5, size=(len(names), 3))
        (d / "poses.txt").write_text("".join(f"{n} " + " ".join(f"{v:.6f}" for v in np.r_[q[i], t[i]]) + "\n"
                                             for i, n in enumerate(names)))
    zp = root / "submission.zip"
    with zipfile.ZipFile(zp, "w") as zf:
        for s in range(scenes):
            lines = []
            for i in range(frames):
                q = rng.normal(size=4)
                lines.append(f"seq1/frame_{i:05d}.jpg " + " ".join(f"{v:.6f}" for v in np.r_[q / np.linalg.norm(q),
                             rng.uniform(-1.5, 1.5, 3)]) + f" {rng.integers(0, 500)}")
            zf.writestr(f"pose_s{s:05d}.txt", "\n".join(lines))
    return zp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=65)
    ap.add_argument("--graded", type=int, default=115, help="graded frames per scene")
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()

    import logging
    import torch
    from mickey_b200 import mapfree_eval as mfe
    from oracle import mapfree_eval_oracle as orc
    assert torch.cuda.is_available(), "this benchmark times the GPU kernel and needs a CUDA device"
    logging.disable(logging.WARNING)
    with tempfile.TemporaryDirectory() as tmp:
        zp = write_split(Path(tmp), args.scenes, args.graded)
        # the graded frames, collected as the evaluator collects them
        with zipfile.ZipFile(zp) as zf:
            fr = [mfe._scene_frames(Path(tmp) / "val", zf, f"s{s:05d}")[0] for s in range(args.scenes)]
        host = [np.concatenate([f[k] for f in fr]) for k in ("q_est", "t_est", "q_gt", "t_gt", "K")]
        P = len(host[0])
        dev = [torch.from_numpy(a).cuda() for a in host]
        out = mfe.frame_metrics_dev(*dev, 540, 720)
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
        for a, b in ev:
            a.record()
            mfe.frame_metrics_dev(*dev, 540, 720, out=out)
            b.record()
        torch.cuda.synchronize()
        kernel_us = float(np.median([a.elapsed_time(b) for a, b in ev]) * 1e3)

        t0 = time.perf_counter()
        metrics, _ = mfe.evaluate_submission(Path(tmp), zp, "val")
        eval_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        r = subprocess.run([sys.executable, "-m", "mickey_b200.mapfree_eval", "--submission_path", str(zp), "--split",
                            "val", "--dataset_path", tmp, "--log", "error"], capture_output=True, text=True, cwd=ROOT)
        cli_s = time.perf_counter() - t0
        assert r.returncode == 0, r.stderr[-2000:]
        assert json.loads(r.stdout) == metrics

        t0 = time.perf_counter()
        ref = orc.frame_metrics(*host, 540, 720)
        oracle_s = time.perf_counter() - t0
        got = out.cpu().numpy()
        max_rel = float(np.max(np.abs(got[:, [0, 2]] - ref[:, [0, 2]]) / np.abs(ref[:, [0, 2]])))

    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(), "power_limit": power, "scenes": args.scenes, "frames": P,
                      "kernel_us": kernel_us, "evaluate_submission_s": eval_s, "cli_process_s": cli_s,
                      "oracle_host_s": oracle_s, "max_rel_diff_trans_reproj": max_rel}))


if __name__ == "__main__":
    main()
