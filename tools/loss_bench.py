"""Time one MetricPoseLoss step at the released training config: mickey_b200.loss.MetricPoseLoss (CUDA search and
gradient, autograd tail) against the reference's algorithm in eager torch (oracle/loss_oracle.py in fp32, which tiles
final_scores to [B*IM, N*N] for torch.multinomial and assembles the gradient in a loop over the B*IM iterations, as
loss_class.py:136-261 does).

    python tools/loss_bench.py [--batch 8] [--reps 5]

Workload: B = 8 pairs at 720x540 (N = 1938 keypoints), IT_MATCHES = IT_RANSAC = 20, 512 samples, 8-point hypotheses,
4 refinements (curriculum_learning.yaml:55-87).  final_scores is a seeded random matrix whose rows concentrate like a
dual softmax's; kps / depths are seeded random.  A step is forward + avg_loss.backward(), timed with CUDA events after
a warm-up.  Prints one JSON line with the card name and its power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mickey_b200.loss import LossParams, MetricPoseLoss  # noqa: E402
from oracle import loss_oracle  # noqa: E402
from tests import loss_cases  # noqa: E402


def smi(field):
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={field}",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def batch(B, N=1938, seed=0):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, N, N, generator=g) * 3.0
    fs = torch.softmax(logits, 1) * torch.softmax(logits, 2)
    K = torch.tensor([[700.0, 0, 270], [0, 700.0, 360], [0, 0, 1]]).repeat(B, 1, 1)
    T = loss_cases.planted_pose().float().unsqueeze(0).repeat(B, 1, 1)
    b = {"final_scores": fs, "kps0": torch.rand(B, 2, N, generator=g) * 540, "kps1": torch.rand(B, 2, N, generator=g) * 540,
         "depth_kp0": 1 + 4 * torch.rand(B, 1, N, generator=g), "depth_kp1": 1 + 4 * torch.rand(B, 1, N, generator=g),
         "K_color0": K, "K_color1": K.clone(), "Kori_color0": K.clone(), "Kori_color1": K.clone(), "T_0to1": T}
    return {k: v.cuda() for k, v in b.items()}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return sorted(ms)[len(ms) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_bench needs a CUDA device")
    cfg = loss_cases.loss_cfg(it_matches=20, it_ransac=20, topk=True)
    p = LossParams(cfg)
    data = batch(a.batch)
    loss = MetricPoseLoss(cfg)

    def ours():
        avg, _, grads, _ = loss(data)
        avg.backward()
        return grads

    def eager():
        r = loss_oracle.metric_pose_loss(data, p, dtype=torch.float32)
        r["avg_loss"].backward()
        return r["probs_grad"]

    t_ours = timed(ours, a.reps)
    t_eager = timed(eager, a.reps)
    print(json.dumps({"card": torch.cuda.get_device_name(), "power_limit": smi("power.limit"), "B": a.batch, "N": 1938,
                      "it_matches": p.it_matches, "it_ransac": p.it_ransac, "n_sample": p.n_sample, "n_corr": p.num_corr,
                      "ms_cuda": round(t_ours, 3), "ms_eager": round(t_eager, 3), "speedup": round(t_eager / t_ours, 2)}))


if __name__ == "__main__":
    main()
