"""Time the training loss's differentiable tail both ways: autograd (MetricPoseLoss's default) against CUDA
(MetricPoseLoss(cfg, cuda_tail=True), csrc/loss_tail.cu).

    python tools/loss_tail_bench.py [--reps 7] [--iters 10] [--out DIR]

Two workloads, the reference's two training shapes:
- curriculum: B = 8 pairs at 720x540 (N = 1938), IT_MATCHES = IT_RANSAC = 20, 512 samples, null hypothesis, top-K
  (curriculum_learning.yaml);
- warm-up: B = 24 pairs at 480x360 (N = 850), IT_MATCHES = IT_RANSAC = 20, 64 samples, no null hypothesis
  (curriculum_learning_warm_up.yaml).
final_scores is a seeded random matrix whose rows concentrate like a dual softmax's; kps / depths are seeded random
(tools/loss_bench.py's batch).  For each workload and variant:
- tail: the tail alone from one fixed search (forward, then backward of loss_value / loss_rot / loss_trans with fixed
  upstream gradients into the kps / depth leaves);
- loss: the whole MetricPoseLoss forward plus avg_loss.backward();
- peak memory of one tail (forward + backward) and of one loss step above what was allocated before it.
Timings are CUDA events around `iters` back-to-back calls, `reps` windows per variant with the two variants alternating;
the JSON line reports the median and the range over windows, the card's name and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mickey_b200.loss import LossParams, MetricPoseLoss, _loss_search_bits, unpack_mask  # noqa: E402
from tests import loss_cases  # noqa: E402
from tools.loss_bench import batch as make_batch, smi  # noqa: E402

WORKLOADS = {
    "curriculum": dict(B=8, N=1938, cfg=lambda: loss_cases.loss_cfg(it_matches=20, it_ransac=20, topk=True)),
    "warm_up": dict(B=24, N=850, cfg=lambda: loss_cases.reference_cfg("curriculum_learning_warm_up")),
}


def tail_fn(loss, data, cuda):
    """One tail, forward and backward, from a fixed search."""
    p = loss.p
    leaves = [data[k].detach().clone().requires_grad_() for k in ("kps0", "depth_kp0", "kps1", "depth_kp1")]
    K0, K1 = data["K_color0"].float(), data["K_color1"].float()
    sampled, _, bits, status = _loss_search_bits(data["final_scores"], *leaves[:2], *leaves[2:], K0, K1, p, 1234)
    assert status == 0, status
    B, N = data["final_scores"].shape[:2]
    Rgt, tgt = data["T_0to1"][:, :3, :3], data["T_0to1"][:, :3, 3:].transpose(1, 2)
    g = torch.Generator(device=K0.device).manual_seed(5)
    ups = [torch.randn(B * p.it_matches, device=K0.device, generator=g) for _ in range(3)]
    inl = unpack_mask(bits, p.n_sample)

    def run():
        for t in leaves:
            t.grad = None
        if cuda:
            out = loss._cuda_tail(data, sampled, bits, *leaves, K0, K1)
        else:
            out = loss._tail(data, sampled, inl, *leaves, K0, K1, Rgt, tgt, B, N)
        torch.autograd.backward(out, ups)
    return run


def loss_fn(loss, data):
    def run():
        avg, _, _, nv = loss(data, seed=99)
        assert nv == 1
        avg.backward()
    return run


def window(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def peak_above(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def summary(ms):
    s = sorted(ms)
    return {"median_ms": round(s[len(s) // 2], 4), "min_ms": round(s[0], 4), "max_ms": round(s[-1], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for loss_tail_bench.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loss_tail_bench needs a CUDA device")
    result = {"card": torch.cuda.get_device_name(), "power_limit": smi("power.limit"), "reps": a.reps, "iters": a.iters}
    for name, w in WORKLOADS.items():
        cfg = w["cfg"]()
        p = LossParams(cfg)
        data = make_batch(w["B"], w["N"])
        losses = {v: MetricPoseLoss(cfg, cuda_tail=v == "cuda") for v in ("autograd", "cuda")}
        fns = {("tail", v): tail_fn(losses[v], data, v == "cuda") for v in losses}
        fns.update({("loss", v): loss_fn(losses[v], data) for v in losses})
        mem = {f"{what}_{v}": peak_above(fn) for (what, v), fn in fns.items()}
        for fn in fns.values():                           # warm-up: module loads, allocator, cuBLAS / cuSOLVER choices
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        for r in range(a.reps):
            for what in ("tail", "loss"):
                order = ("autograd", "cuda") if r % 2 == 0 else ("cuda", "autograd")
                for v in order:
                    times[(what, v)].append(window(fns[(what, v)], a.iters))
        res = {"B": w["B"], "N": w["N"], "n_sample": p.n_sample, "it_matches": p.it_matches, "it_ransac": p.it_ransac,
               "loss": p.loss_type}
        for (what, v), ms in times.items():
            res[f"{what}_{v}"] = summary(ms)
        for what in ("tail", "loss"):
            res[f"{what}_speedup"] = round(res[f"{what}_autograd"]["median_ms"] / res[f"{what}_cuda"]["median_ms"], 2)
        res["peak_bytes_above_inputs"] = mem
        result[name] = res
        del data, fns, losses
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "loss_tail_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
