"""Time the training model's validation pose solver: mickey_b200.procrustes against the reference's vectorized solver.

    python tools/validation_bench.py [--rounds 5] [--reps 3] [--out result.json]

The model is the recorded MicKeyTrainingModel tree (ViT-L, fp16 backbone) moved onto the CUDA modules by
use_cuda_modules, with seeded synthetic weights and images, at the two validation shapes of the shipped configs:
B = 8 at 720x540 (curriculum_learning) and B = 24 at 480x360 (curriculum_learning_warm_up), PROCRUSTES 20 x 100
hypotheses over 2048 sampled matches.  Two solvers:
    cuda    mickey_b200.procrustes.e2eProbabilisticProcrustesSolver (mk_procrustes_solve)
    eager   oracle/mickey_oracle.py's solve_pose in fp32 torch on the GPU.  It stands in for the reference's
            estimate_pose_vectorized (probabilisticProcrustes.py:183-348): the same algorithm with the same tensors, the
            [B * IT_MATCHES, N * N] copy of final_scores for torch.multinomial (mickey_oracle.py:358, reference :230) and
            the [B * IT_MATCHES * IT_RANSAC, 2048, 3] point sets of the soft inlier count included.
For each: CUDA-event time of one estimate_pose_vectorized call on the validation batch; of a whole validation_step
(model.py:66-89: eval-mode forward of both images, the loss, the solver); and the peak allocation of the solver call above
what was allocated before it (the inputs).  Everything runs under torch.inference_mode, Lightning's default for
validation.  Every shape is warmed up, the two solvers alternate round by round, and the median and the range over all
calls are reported with the card's name and power limit read in the same run.  Needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mickey_b200.procrustes import e2eProbabilisticProcrustesSolver  # noqa: E402
from mickey_b200.training import use_cuda_modules  # noqa: E402
from oracle import mickey_oracle as mo  # noqa: E402
from tests.test_gpu_heads_training import converted_model, step_batch  # noqa: E402
from tests.test_gpu_training_lifecycle import forward_pair, is_eval_model, loss_batch  # noqa: E402

CONFIGS = {"b8_720x540": ("curriculum_learning", 8, 720, 540), "b24_480x360": ("curriculum_learning_warm_up", 24, 480, 360)}


class EagerSolver:
    """The reference solver's computation, restated by the oracle, in fp32 on the batch's device."""

    def __init__(self, cfg):
        self.cfg = cfg

    def estimate_pose_vectorized(self, batch, return_inliers=False):
        d = {k: batch[k].detach() for k in ("final_scores", "kps0", "kps1", "depth_kp0", "depth_kp1", "K_color0", "K_color1")}
        return mo.solve_pose(d["final_scores"], d["kps0"], d["depth_kp0"], d["kps1"], d["depth_kp1"], d["K_color0"].float(),
                             d["K_color1"].float(), self.cfg, return_inliers=return_inliers)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def validation_step(model, solver, ims, data):
    """validation_step (model.py:66-89) with `solver` as e2e_Procrustes."""
    is_eval_model(model, True)
    _, cs, final = forward_pair(model, ims)
    batch = loss_batch(data, cs, final)
    avg_loss, outputs, _, _ = model.loss_fn(batch)
    R, t, inl = solver.estimate_pose_vectorized(batch)[:3]
    return avg_loss, R, t, inl


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("validation_bench needs a CUDA device")
    result = {"card": card(), "configs": {}}
    for cname, (config, B, H, W) in CONFIGS.items():
        torch.manual_seed(0)
        model = use_cuda_modules(converted_model(config), solver=True)
        solvers = {"cuda": model.e2e_Procrustes, "eager": EagerSolver(model.cfg)}
        ims, data = step_batch(B, H, W, seed=B)
        with torch.inference_mode():
            is_eval_model(model, True)
            _, cs, final = forward_pair(model, ims)
            batch = loss_batch(data, cs, final)
            for s in solvers.values():                                   # warm-up of every shape
                s.estimate_pose_vectorized(batch)
                validation_step(model, s, ims, data)
            torch.cuda.synchronize()
            solve_ms = {v: [] for v in solvers}
            step_ms = {v: [] for v in solvers}
            peak = {v: 0 for v in solvers}
            for _ in range(a.rounds):
                for v, s in solvers.items():
                    for _ in range(a.reps):
                        torch.cuda.synchronize()
                        base = torch.cuda.memory_allocated()
                        torch.cuda.reset_peak_memory_stats()
                        ms, _ = timed(lambda: s.estimate_pose_vectorized(batch))
                        peak[v] = max(peak[v], torch.cuda.max_memory_allocated() - base)
                        solve_ms[v].append(ms)
                        step_ms[v].append(timed(lambda: validation_step(model, s, ims, data))[0])
        N = final.shape[-1]
        result["configs"][cname] = {
            "B": B, "N": N, "tile_gb": B * 20 * N * N * 4 / 2 ** 30,
            **{v: {"solve_ms": stats(solve_ms[v]), "validation_step_ms": stats(step_ms[v]),
                   "solve_peak_mb_above_inputs": peak[v] / 2 ** 20} for v in solvers}}
        del model, batch, final, cs
        torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
