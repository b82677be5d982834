"""Time the training backbone (mickey_b200.dinov2.DinoVisionTransformer.forward_features) against a plain-torch fp16
stand-in, and its channel-major final-norm kernel alone against its HBM lower bound.

    python tools/backbone_bench.py [--iters 10] [--warmup 3] [--json OUT]

Shapes: ViT-L with B = 8 at 720x540 (714x532 after the extractor's crop), ViT-L with B = 24 at 476x350 (the warm-up
crop), ViT-B with B = 8 at 720x540.  Weights are the seeded synthetic ones (the timing does not depend on their values).

The stand-in is NOT the reference: the reference runs DINOv2 in fp16 with xformers' memory-efficient attention, and its
tree is not importable here.  It restates the backbone with oracle/mickey_oracle.py's functions on fp16 weights, with
F.scaled_dot_product_attention in place of the eager softmax, followed by the extractor's
permute / reshape / float (mickey_extractor.py:49-51).

Times are CUDA-event times over `iters` calls after `warmup` calls, ours and the stand-in alternating.  Peak memory is
torch.cuda.max_memory_allocated during one call minus what was allocated before it (inputs and module parameters); ours
is measured on a cold module, so it includes the packed weights and the workspace.  The final norm
is timed by the library's per-kernel events (mk_profile_enable) over the same calls.  The card's name, power limit and
maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mickey_b200.config import VARIANTS, mickey_cfg  # noqa: E402
from mickey_b200.dinov2 import DinoVisionTransformer  # noqa: E402
from mickey_b200.weights import BACKBONE, synthetic_state_dict  # noqa: E402
from oracle import mickey_oracle as mo  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
SHAPES = [("vitl", 8, 714, 532, "720x540"), ("vitl", 24, 476, 350, "476x350 (warm-up)"), ("vitb", 8, 714, 532, "720x540")]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.stdout else None}


def standin(sd16, x, heads, depth):
    """fp16 torch restatement of forward_features + the extractor's layout change (stand-in for fp16 + xformers)."""
    t = mo.vit_tokens(sd16, x)
    B, T, D = t.shape
    for i in range(depth):
        p = f"{BACKBONE}blocks.{i}."
        h = F.layer_norm(t, (D,), sd16[p + "norm1.weight"], sd16[p + "norm1.bias"], eps=1e-6)
        qkv = F.linear(h, sd16[p + "attn.qkv.weight"], sd16[p + "attn.qkv.bias"]).reshape(B, T, 3, heads, 64).permute(2, 0, 3, 1, 4)
        a = F.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2]).transpose(1, 2).reshape(B, T, D)
        t = t + sd16[p + "ls1.gamma"] * F.linear(a, sd16[p + "attn.proj.weight"], sd16[p + "attn.proj.bias"])
        h = F.layer_norm(t, (D,), sd16[p + "norm2.weight"], sd16[p + "norm2.bias"], eps=1e-6)
        t = t + sd16[p + "ls2.gamma"] * mo.vit_mlp(sd16, p + "mlp.", h)
    t = F.layer_norm(t, (D,), sd16[BACKBONE + "norm.weight"], sd16[BACKBONE + "norm.bias"], eps=1e-6)[:, 1:]
    gh, gw = x.shape[-2] // 14, x.shape[-1] // 14
    return t.permute(0, 2, 1).reshape(B, D, gh, gw).float()


def timed(fn, iters):
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def peak_above(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return peak


def profile_tag(m, tag):
    lib, h = m._packed.lib, m._packed.h
    import ctypes as C
    buf = C.create_string_buffer(1 << 16)
    assert lib.mk_profile_read(h, buf, len(buf)) == 0
    for line in buf.value.decode().splitlines():
        name, n, ms = line.split()
        if name == tag:
            return int(n), float(ms)
    raise RuntimeError(f"no '{tag}' launches were profiled")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("backbone_bench.py measures on a CUDA device; none is available")
    res = {"card": card(), "iters": args.iters, "warmup": args.warmup, "rows": []}
    for variant, B, H, W, label in SHAPES:
        D, depth, heads = VARIANTS[variant]
        sd = {k: v for k, v in synthetic_state_dict(mickey_cfg(variant, 2, 8), seed=0).items() if k.startswith(BACKBONE)}
        m = DinoVisionTransformer(variant)
        m.load_state_dict({k[len(BACKBONE):]: v for k, v in sd.items()})
        m = m.cuda().to(torch.float16)
        sd16 = {k: v.cuda().half() for k, v in sd.items()}
        del sd
        x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(0)).cuda().half()
        ours = lambda: m.forward_features(x)["x_norm_patchtokens"]                        # noqa: E731
        ref = lambda: standin(sd16, x, heads, depth)                                      # noqa: E731
        with torch.no_grad():
            for _ in range(args.warmup):
                ours(), ref()
            t_ours, t_ref = [], []
            for _ in range(args.iters):                                                  # alternate the two
                t_ours += timed(ours, 1)
                t_ref += timed(ref, 1)
            pk_ref = peak_above(ref)
            m._packed = None                    # ours from a cold module: the packed weights and the workspace count
            torch.cuda.empty_cache()
            pk_ours = peak_above(ours)
            m._packed.lib.mk_profile_enable(m._packed.h, 1)
            for _ in range(args.iters):
                ours()
            n_ln, ms_ln = profile_tag(m, "vit.layernorm_cm")
            m._packed.lib.mk_profile_enable(m._packed.h, 0)
        N = (H // 14) * (W // 14)
        ln_bytes = B * (N + 1) * D * 4 + B * N * D * 4
        ln_us = ms_ln / n_ln * 1e3
        row = {"variant": variant, "B": B, "image": label, "H": H, "W": W,
               "ours_ms_median": statistics.median(t_ours), "ours_ms_min": min(t_ours),
               "standin_ms_median": statistics.median(t_ref), "standin_ms_min": min(t_ref),
               "ours_peak_mb_above_inputs": pk_ours / 1e6, "standin_peak_mb_above_inputs": pk_ref / 1e6,
               "final_norm_us": ln_us, "final_norm_bytes": ln_bytes,
               "final_norm_hbm_bound_us": ln_bytes / HBM_BYTES_PER_S * 1e6}
        row["speedup"] = row["standin_ms_median"] / row["ours_ms_median"]
        row["final_norm_share_of_bound"] = row["final_norm_hbm_bound_us"] / ln_us
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
        del m, sd16, x
        torch.cuda.empty_cache()
    print(f"\ncard: {res['card']}")
    print(f"{'shape':34s} {'ours ms':>9s} {'torch fp16 ms':>14s} {'x':>6s} {'ours MB':>9s} {'torch MB':>9s} "
          f"{'norm us':>8s} {'bound us':>9s}")
    for r in res["rows"]:
        print(f"{r['variant'] + ' B=' + str(r['B']) + ' ' + r['image']:34s} {r['ours_ms_median']:9.2f} "
              f"{r['standin_ms_median']:14.2f} {r['speedup']:6.2f} {r['ours_peak_mb_above_inputs']:9.0f} "
              f"{r['standin_peak_mb_above_inputs']:9.0f} {r['final_norm_us']:8.1f} {r['final_norm_hbm_bound_us']:9.1f}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
