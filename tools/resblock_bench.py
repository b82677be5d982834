"""Time the heads' residual block, forward + backward in train mode, against eager torch (cuDNN) on the same GPU.

    python tools/resblock_bench.py [--reps 12] [--warmup 3] [--out results.json]
    python tools/resblock_bench.py --split     # per contraction and per kernel, wide blocks at both shapes

Shapes: the two training configurations, B = 8 at 51 x 38 (curriculum / overlap, 720 x 540) and B = 24 at 34 x 25
(warm-up, 476 x 350).  For each, the five block shapes (1024->512, 512->256, 256->128, 128->64, 128->128), then all 16
blocks of one extractor call (four heads of rb1..rb4; three heads end in 128->64, the descriptor head in 128->128 without
the final ReLU).  rb1's input comes from the frozen backbone and needs no gradient, as in training.

The comparison is the same block written with torch.nn.functional (conv2d, batch_norm in train mode, relu) run as eager
fp32 autograd under torch's default flags, so cuDNN computes the convolutions in TF32.  The two alternate; each reports
the median and spread of CUDA-event times after warm-up, the peak max_memory_allocated above the inputs, and the TFLOP/s
reached on the convolution FLOPs derived from the shapes (forward, weight gradients, data gradients; rb1 takes no data
gradient).  The card's name and power limit are read in the same run.
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
import ctypes as C  # noqa: E402

from mickey_b200 import _lib  # noqa: E402
from mickey_b200.resblock import BasicBlock  # noqa: E402

GEOMS = [(8, 38, 51), (24, 25, 34)]
BLOCKS = [(1024, 512), (512, 256), (256, 128), (128, 64), (128, 128)]
HEAD = {"kp": [(1024, 512, True), (512, 256, True), (256, 128, True), (128, 64, True)],
        "dsc": [(1024, 512, True), (512, 256, True), (256, 128, True), (128, 128, False)]}
EXTRACTOR = HEAD["kp"] * 3 + HEAD["dsc"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def flops(cin, cout, M, dgrad):
    """Convolution FLOPs of one block's forward + backward over M = B h w pixels."""
    fwd = 2 * M * cout * (9 * cin + 9 * cout + (cin if cin != cout else 0))
    conv2_dgrad = 2 * M * cout * 9 * cout
    first_dgrad = 2 * M * cout * (9 * cin + (cin if cin != cout else 0)) if dgrad else 0
    return 2 * fwd + conv2_dgrad + first_dgrad


def eager(m, x, relu):
    def bn(z, b):
        return F.batch_norm(z, b.running_mean, b.running_var, b.weight, b.bias, True, b.momentum, b.eps)
    a1 = F.relu(bn(F.conv2d(x, m.conv1.weight, padding=1), m.bn1))
    out = bn(F.conv2d(a1, m.conv2.weight, padding=1), m.bn2)
    out = out + (F.conv2d(x, m.shortcut[0].weight) if hasattr(m, "shortcut") else x)
    return F.relu(out) if relu else out


def time_pair(steps, reps, warmup):
    times = {k: [] for k in steps}
    peak = {}
    for name, fn in steps.items():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        for _ in range(warmup):
            fn()
    for _ in range(reps):
        for name, fn in steps.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e))
    return {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "peak_mb": peak[k]}
            for k, v in times.items()}


def run_set(specs, B, h, w, reps, warmup):
    """specs: [(cin, cout, relu, input_needs_grad)]; runs them one after another as one step."""
    dev = "cuda"
    torch.manual_seed(0)
    mods = [BasicBlock(ci, co).to(dev) for ci, co, _, _ in specs]
    xs = [torch.randn(B, ci, h, w, device=dev) for ci, _, _, _ in specs]
    gos = [torch.randn(B, co, h, w, device=dev) for _, co, _, _ in specs]

    def step(fn):
        def go():
            for m, x, g, (_, _, relu, need) in zip(mods, xs, gos, specs):
                xx = x.detach().requires_grad_(need)
                fn(m, xx, relu).backward(g)
                m.zero_grad(set_to_none=True)
        return go
    res = time_pair({"cuda": step(lambda m, x, r: m(x, relu=r)), "eager": step(eager)}, reps, warmup)
    fl = sum(flops(ci, co, B * h * w, need) for ci, co, _, need in specs)
    for v in res.values():
        v["tflops"] = fl / (v["median_ms"] * 1e-3) / 1e12
    res["tflop"] = fl / 1e12
    res["speedup"] = res["eager"]["median_ms"] / res["cuda"]["median_ms"]
    return res


def _events(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return statistics.median(ts)


def split(reps, warmup):
    """Each convolution contraction of a block alone, ours (mk_op_conv_tf32, including its per-call weight re-layout and,
    for the weight gradient, the per-tap shifted copies and the slot fold) against cuDNN's (conv2d, conv2d_input,
    conv2d_weight under default TF32 flags); then a torch.profiler breakdown of one block's forward + backward by kernel."""
    lib = _lib.load()
    dev = "cuda"
    stream = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for B, h, w in GEOMS:
        for cin, cout in ((1024, 512), (512, 256)):
            R = B * (h + 2) * (w + 2)
            Rp = (R + 3) // 4 * 4
            M = B * h * w
            x = torch.randn(B, cin, h, w, device=dev)
            dz = torch.randn(B, cout, h, w, device=dev)
            W = torch.randn(cout, cin, 3, 3, device=dev) * 0.02
            xp = torch.randn(R, cin, device=dev)
            dzp = torch.randn(R, cout, device=dev)
            dzT, xT = torch.randn(cout, Rp, device=dev), torch.randn(cin, Rp, device=dev)
            outs = {0: torch.empty(R, cout, device=dev), 1: torch.empty(R, cin, device=dev), 2: torch.empty_like(W)}
            args = {0: (xp, W), 1: (dzp, W), 2: (dzT, xT)}
            row = {"B": B, "h": h, "w": w, "conv": f"3x3 {cin}->{cout}", "gflop": 2 * M * cout * 9 * cin / 1e9}
            theirs = {0: lambda: F.conv2d(x, W, padding=1),
                      1: lambda: torch.nn.grad.conv2d_input(x.shape, W, dz, padding=1),
                      2: lambda: torch.nn.grad.conv2d_weight(x, W.shape, dz, padding=1)}
            for mode, name in ((0, "forward"), (1, "dgrad"), (2, "wgrad")):
                nb = int(lib.mk_op_conv_tf32_ws_bytes(mode, B, h, w, cin, cout, 9))
                ws = torch.empty(nb, dtype=torch.uint8, device=dev)
                a, b = args[mode]
                ours = lambda: _lib.check(lib.mk_op_conv_tf32(mode, _lib.ptr(a), _lib.ptr(b), _lib.ptr(outs[mode]), B, h, w,
                                                              cin, cout, 9, _lib.ptr(ws), nb, stream()), "conv")
                row[name] = {"cuda_ms": _events(ours, reps, warmup), "cudnn_ms": _events(theirs[mode], reps, warmup)}
            print(json.dumps(row), flush=True)
        # per kernel, one 1024->512 block, forward + backward, rb1 without dX
        m = BasicBlock(1024, 512).to(dev)
        x = torch.randn(B, 1024, h, w, device=dev)
        go = torch.randn(B, 512, h, w, device=dev)
        step = lambda: (m(x).backward(go), m.zero_grad(set_to_none=True))
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                step()
            torch.cuda.synchronize()
        tot = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" or getattr(ev, "self_device_time_total", 0):
                t = getattr(ev, "self_device_time_total", None) or getattr(ev, "self_cuda_time_total", 0)
                key = ev.key.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0][:90]
                tot[key] = tot.get(key, 0) + t / reps / 1000.0
        top = sorted(tot.items(), key=lambda kv: -kv[1])[:14]
        print(json.dumps({"B": B, "h": h, "w": w, "block": "1024->512 per kernel (ms per step)",
                          "kernels": {k: round(v, 3) for k, v in top}, "total_ms": round(sum(tot.values()), 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--split", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    if a.split:
        print(json.dumps({"card": card()}))
        split(a.reps, a.warmup)
        return
    res = {"card": card(), "rows": []}
    for B, h, w in GEOMS:
        for cin, cout in BLOCKS:
            r = run_set([(cin, cout, (cin, cout) != (128, 128), cin != 1024)], B, h, w, a.reps, a.warmup)
            row = {"B": B, "h": h, "w": w, "block": f"{cin}->{cout}", **r}
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
        specs = [(ci, co, relu, ci != 1024) for ci, co, relu in EXTRACTOR]
        r = run_set(specs, B, h, w, a.reps, a.warmup)
        row = {"B": B, "h": h, "w": w, "block": "extractor (16 blocks)", **r}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": res["card"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
