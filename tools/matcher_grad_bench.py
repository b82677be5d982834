"""Time the matcher's training chain, forward + backward, against the reference's eager fp32 autograd on the same GPU.

    python tools/matcher_grad_bench.py [--reps 10] [--warmup 3] [--out results.json]

Chain: scores (dual-softmax with the dustbin), kp_scores, final_scores = scores * kp_scores, log(final + 1e-16) and the
backward with a REINFORCE-shaped sparse probs_grad (512 cells drawn per set, 20 sets per pair), at the released training
shape (B = 8, 720 x 540, N = 1938) and the warm-up shape (B = 24, 480 x 360, N = 850).  The reference side restates
feature_matcher.py:64-83 + compute_correspondences.py:46-50 + model.py:201 in torch.  The two implementations alternate;
each reports the median of CUDA-event times after warm-up and its peak torch.cuda.max_memory_allocated.  The card's name
and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mickey_b200.dual_softmax import dual_softmax  # noqa: E402

SHAPES = [(8, 1938), (24, 850)]
T = 0.1


def reference_chain(d0, d1, alpha, s0, s1):
    s = torch.matmul(d0.transpose(1, 2).contiguous(), d1) / T
    b, m, n = s.shape
    bins0, bins1, a = alpha.expand(b, m, 1), alpha.expand(b, 1, n), alpha.expand(b, 1, 1)
    c = torch.cat([torch.cat([s, bins0], -1), torch.cat([bins1, a], -1)], 1)
    scores = (F.softmax(c, 1) * F.softmax(c, 2))[:, :-1, :-1]
    kp = torch.matmul(s0.transpose(2, 1).contiguous(), s1)
    return scores * kp


def cuda_chain(d0, d1, alpha, s0, s1):
    return dual_softmax(d0, d1, alpha, T, s0, s1, unit_norm=True)[2]


def inputs(B, N, dev):
    g = torch.Generator(device=dev).manual_seed(B * N)
    d0 = F.normalize(torch.randn(B, 128, N, device=dev, generator=g), dim=1)
    d1 = F.normalize(torch.randn(B, 128, N, device=dev, generator=g), dim=1)
    s0, s1 = torch.rand(B, 1, N, device=dev, generator=g), torch.rand(B, 1, N, device=dev, generator=g)
    pg = torch.zeros(B * N * N, device=dev)
    idx = torch.randint(0, N * N, (B, 20 * 512), device=dev, generator=g) + torch.arange(B, device=dev)[:, None] * N * N
    pg[idx.reshape(-1)] = torch.randn(idx.numel(), device=dev, generator=g)
    return d0, d1, s0, s1, pg.reshape(B, N, N)


def step(chain, d0, d1, s0, s1, pg, alpha):
    leaves = [t.detach().clone().requires_grad_() for t in (d0, d1, s0, s1)]
    a = alpha.detach().clone().requires_grad_()
    fin = chain(leaves[0], leaves[1], a, leaves[2], leaves[3])
    torch.autograd.backward(torch.log(fin + 1e-16), pg)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip() or torch.cuda.get_device_name(dev)
    res = {"card": card, "shapes": []}
    alpha = torch.tensor(1.0, device=dev)
    for B, N in SHAPES:
        d0, d1, s0, s1, pg = inputs(B, N, dev)
        impls = {"cuda": cuda_chain, "reference_eager": reference_chain}
        times = {k: [] for k in impls}
        peak = {}
        for k, f in impls.items():
            for _ in range(a.warmup):
                step(f, d0, d1, s0, s1, pg, alpha)
        for _ in range(a.reps):
            for k, f in impls.items():                         # alternated
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(f, d0, d1, s0, s1, pg, alpha)
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1))
                peak[k] = max(peak.get(k, 0), torch.cuda.max_memory_allocated() - base)
        row = {"B": B, "N": N}
        for k in impls:
            row[k] = {"median_ms": statistics.median(times[k]), "min_ms": min(times[k]), "peak_mb": peak[k] / 2 ** 20}
        res["shapes"].append(row)
        print(json.dumps(row), flush=True)
        del d0, d1, s0, s1, pg
        torch.cuda.empty_cache()
    print(json.dumps({"card": card}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
