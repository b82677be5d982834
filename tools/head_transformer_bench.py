"""Time one call of the heads' transformer, forward + backward, against an eager fp32 torch stand-in on the same GPU.

    python tools/head_transformer_bench.py [--reps 20] [--warmup 5] [--out results.json]

Shapes: the two training configurations, B = 8 at 51 x 38 (curriculum_learning, 720 x 540) and B = 24 at 34 x 25
(warm-up, 476 x 350), 3 layers, with the positional encoding.  The stand-in is the reference module's forward written
with torch.nn.functional: the module's device-resident PE slice added to the input, then oracle.mickey_oracle.encoder_layer
three times, run as eager fp32 autograd with TF32 off, as the reference trains; the reference module itself is not used.
Both compute dX and every parameter gradient.  The two alternate; each reports the median and spread of CUDA-event times after warm-up and its peak max_memory_allocated above
the inputs.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mickey_b200.head_transformer import Transformer_self_att  # noqa: E402
from oracle import mickey_oracle as mo  # noqa: E402

SHAPES = [(8, 38, 51), (24, 25, 34)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda"
    res = {"card": card(), "shapes": []}
    for B, h, w in SHAPES:
        torch.manual_seed(0)
        m = Transformer_self_att(128, 3, True).to(dev)
        with torch.no_grad():
            for l in m.layers:
                for n in (l.norm1, l.norm2):
                    n.weight.add_(0.1 * torch.randn_like(n.weight))
        x = torch.randn(B, 128, h, w, device=dev)
        go = torch.randn(B, 128, h, w, device=dev)
        sd = {f"att.layers.{i}.{k}": v for i, l in enumerate(m.layers) for k, v in l.state_dict().items()}
        sd = {k: v.detach().clone().requires_grad_() for k, v in sd.items()}

        def cuda_step():
            xx = x.detach().requires_grad_()
            m(xx).backward(go)
            m.zero_grad(set_to_none=True)

        pe = m.posEnc.pe[:, :, :h, :w]          # the module's device buffer, as the reference module adds it

        def eager_step():
            xx = x.detach().requires_grad_()
            t = (xx + pe).flatten(2).transpose(1, 2)
            for i in range(3):
                t = mo.encoder_layer(sd, f"att.layers.{i}.", t)
            t.transpose(1, 2).reshape(B, 128, h, w).backward(go)
            for v in sd.values():
                v.grad = None

        times = {"cuda": [], "eager": []}
        peak = {}
        for name, fn in (("cuda", cuda_step), ("eager", eager_step)):
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            fn()
            torch.cuda.synchronize()
            peak[name] = torch.cuda.max_memory_allocated() - base
            for _ in range(a.warmup):
                fn()
        for _ in range(a.reps):
            for name, fn in (("cuda", cuda_step), ("eager", eager_step)):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn()
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e))
        T = B * h * w
        row = {"B": B, "h": h, "w": w, "tokens": T, "gflop": 3 * T * (327680 + 655360) / 1e9}
        for name in times:
            t = sorted(times[name])
            row[name] = {"median_ms": statistics.median(t), "min_ms": t[0], "max_ms": t[-1],
                         "peak_mb": peak[name] / 2 ** 20}
        row["speedup"] = row["eager"]["median_ms"] / row["cuda"]["median_ms"]
        res["shapes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": res["card"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
