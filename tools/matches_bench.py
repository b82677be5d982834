"""Time mk_mutual_matches (MicKey's correspondences, featureMatcher.get_matches_list in CUDA) on the engine's own
final_scores, and the same list computed by eager PyTorch on the GPU pair by pair (oracle/matches_oracle.py, the
restatement of the reference's get_matches_list):

    python tools/matches_bench.py [--iters 50] [--warmup 10]

C2: one 720x540 ViT-S pair; C3: 32 720x540 ViT-B pairs.  final_scores is the engine's padded [B, N, 1952][:, :, :N] view.
GB/s counts the (N-1) x (N-1) candidate cells read once per pair.  Prints one JSON line per case, with the card name and
its power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mickey_b200.config import mickey_cfg                      # noqa: E402
from mickey_b200.matches import mutual_matches_raw             # noqa: E402
from mickey_b200.model import build_model                      # noqa: E402
from mickey_b200.weights import synthetic_checkpoint           # noqa: E402
from oracle.matches_oracle import matches_list                 # noqa: E402
from tests.common import synthetic_pair                        # noqa: E402


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={fields}",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10)
        return r.stdout.strip() if r.returncode == 0 else "n/a"
    except (OSError, subprocess.TimeoutExpired):
        return "n/a"


def time_us(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    os.environ.setdefault("MICKEY_SYNTHETIC_BACKBONE", "1")
    card = {"card": torch.cuda.get_device_name(), "power_limit_W": smi("power.limit")}
    for name, variant, it_m, it_r, B in (("c2", "vits", 8, 64, 1), ("c3", "vitb", 16, 64, 32)):
        cfg = mickey_cfg(variant, it_m, it_r)
        model = build_model(cfg, synthetic_checkpoint(cfg, seed=0, with_backbone=True))
        model.static_outputs = True                     # data["final_scores"] is the engine's padded buffer itself
        data = {k: v.cuda() for k, v in synthetic_pair(B, 720, 540, seed=0).items()}
        torch.manual_seed(0)
        model(data)
        fs = data["final_scores"]
        N = fs.shape[-1]
        us = time_us(lambda: mutual_matches_raw(fs), a.iters, a.warmup)
        eager_iters = max(1, a.iters // 10)
        eager = time_us(lambda: [matches_list(fs[b]) for b in range(B)], eager_iters, 2)
        gb = B * (N - 1) ** 2 * 4 / 1e9
        print(json.dumps({"case": name, "pairs": B, "N": N, "pitch": fs.stride(1), "us_per_call": round(us, 2),
                          "GB_per_s": round(gb / (us * 1e-6), 1), "eager_torch_us_per_call": round(eager, 1),
                          "speedup_vs_eager": round(eager / us, 1), **card}), flush=True)
        del model, data, fs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
