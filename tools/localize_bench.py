"""Queries against one cached reference, six ways, alternated on one GPU:

    (a) forward      model(data) on the explicit pairs (the reference re-extracted for every pair)
    (b) banks        extract_features(queries) + pose_from_features (two eager C calls)
    (c) localize     model.localize, eager
    (d) graph        model.localize, replayed from a CUDA graph
    (e) pipelined    model.localize with pipeline_depth 2, pinned uint8 host frames
    (f) static       (d) with static_outputs: the outputs are the engine's buffers, not clones

    MICKEY_SYNTHETIC_BACKBONE=1 python tools/localize_bench.py --workloads C2,C3 --P 1,4,32 --steps 20 --warmup 3 --runs 3

Workloads: C2 = ViT-S, 512 hypotheses; C3 = ViT-B, 1024 hypotheses; 720x540 images.  Each run times every (P, variant)
once, in order, so the variants alternate.  Per variant it reports ms per step (a window of --steps back-to-back calls
ending in one synchronise), the median latency of one call (synchronised before and after; the single-query latency at
P = 1), and the peak memory the variant's calls allocate.  It also prints one SHA-256 per variant over the R, t, inliers,
kps, depth and final_scores of one seeded call: equal digests are equal outputs.  Writes nothing but stdout (--out: a
JSON file).
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mickey_b200.config import mickey_cfg                          # noqa: E402
from mickey_b200.io import to_float_chw                             # noqa: E402
from mickey_b200.model import MickeyRelativePose                    # noqa: E402
from mickey_b200.weights import synthetic_state_dict                # noqa: E402

WORKLOADS = {"C2": ("vits", 8, 64), "C3": ("vitb", 16, 64)}
VARIANTS = ("a_forward", "b_banks", "c_localize", "d_graph", "e_pipelined", "f_static")
HASH_KEYS = ("R", "t", "inliers", "kps0", "kps1", "depth_kp0", "depth_kp1", "final_scores")
H, W = 720, 540


def _model(cfg, dev, **attrs):
    m = MickeyRelativePose(cfg)
    m.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    m = m.to(dev).eval()
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


def _digest(d):
    h = hashlib.sha256()
    for k in HASH_KEYS:
        h.update(d[k].detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


class Workload:
    def __init__(self, name, P, dev):
        variant, im, ir = WORKLOADS[name]
        cfg = mickey_cfg(variant, im, ir)
        self.P, self.dev = P, dev
        self.eager = _model(cfg, dev, use_graph=False)
        self.graph = _model(cfg, dev)
        self.piped = _model(cfg, dev, pipeline_depth=2)
        self.static = _model(cfg, dev, static_outputs=True)
        g = torch.Generator().manual_seed(1000 + P)
        ref_u8 = torch.randint(0, 256, (1, H, W, 3), generator=g, dtype=torch.uint8)
        q_u8 = torch.randint(0, 256, (P, H, W, 3), generator=g, dtype=torch.uint8)
        self.ref_img = to_float_chw(ref_u8).to(dev)
        self.queries = to_float_chw(q_u8).to(dev)
        self.queries_u8_host = q_u8.pin_memory()
        self.K = torch.tensor([[549.7, 0, 268.7], [0, 549.7, 351.8], [0, 0, 1.0]], device=dev)[None].repeat(P, 1, 1)
        self.K_host = self.K.cpu().pin_memory()
        self.image0 = self.ref_img.expand(P, -1, -1, -1).contiguous()
        # the cached reference of every localize / bank variant, extracted once per model
        self.refs = {id(m): m.extract_features(self.ref_img) for m in (self.eager, self.graph, self.piped, self.static)}
        self.idx = [0] * P

    def step(self, v):
        P = self.P
        if v == "a_forward":
            data = {"image0": self.image0, "image1": self.queries, "K_color0": self.K, "K_color1": self.K}
            self.graph(data)
            return data
        if v == "b_banks":
            m = self.eager
            qb = m.extract_features(self.queries)
            return m.pose_from_features(self.refs[id(m)], self.idx, qb, range(P), self.K, self.K)
        if v == "c_localize":
            m = self.eager
            return m.localize(self.refs[id(m)], self.idx, self.queries, self.K, self.K)
        if v == "d_graph":
            m = self.graph
            return m.localize(self.refs[id(m)], self.idx, self.queries, self.K, self.K)
        if v == "f_static":
            m = self.static
            return m.localize(self.refs[id(m)], self.idx, self.queries, self.K, self.K)
        m = self.piped
        return m.localize(self.refs[id(m)], self.idx, self.queries_u8_host, self.K_host, self.K_host)


def _measure(wl, v, steps, warmup):
    for _ in range(warmup):
        wl.step(v)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    for _ in range(steps):
        wl.step(v)
    torch.cuda.synchronize()
    ms_step = (time.perf_counter() - t0) * 1e3 / steps
    lat = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        wl.step(v)
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t0) * 1e3)
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    return ms_step, statistics.median(lat), peak


def _gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                      # the measurement stands without it; say so
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C2,C3")
    ap.add_argument("--P", default="1,4,32")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write every record to this JSON file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("localize_bench needs a CUDA device (an H100); there is nothing to measure on the CPU")
    os.environ.setdefault("MICKEY_SYNTHETIC_BACKBONE", "1")
    dev = torch.device("cuda", 0)
    gpu = _gpu_info()
    print(json.dumps({"gpu": gpu, "torch": torch.__version__}), flush=True)
    records = []
    for name in args.workloads.split(","):
        for P in map(int, args.P.split(",")):
            wl = Workload(name, P, dev)
            digests = {}
            for v in VARIANTS:
                torch.manual_seed(1234)
                out = wl.step(v)
                torch.cuda.synchronize()
                digests[v] = _digest(out)
            times = {v: [] for v in VARIANTS}
            for run in range(args.runs):
                for v in VARIANTS:
                    times[v].append(_measure(wl, v, args.steps, args.warmup))
            for v in VARIANTS:
                ms = [t[0] for t in times[v]]
                lat = [t[1] for t in times[v]]
                rec = {"workload": name, "P": P, "variant": v, "ms_per_step": ms, "ms_per_step_median": statistics.median(ms),
                       "latency_ms": lat, "latency_ms_median": statistics.median(lat), "peak_mb": max(t[2] for t in times[v]),
                       "sha256": digests[v], "gpu": gpu, "runs": args.runs, "steps": args.steps}
                records.append(rec)
                print(json.dumps(rec), flush=True)
            same = len(set(digests.values())) == 1
            print(json.dumps({"workload": name, "P": P, "outputs_equal": same}), flush=True)
            del wl
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(records, f, indent=1)


if __name__ == "__main__":
    main()
