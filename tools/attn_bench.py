"""Attention kernel timing at the C2 (2 images, 6 heads: ViT-S) and C3 (64 images, 12 heads: ViT-B) shapes.

    python tools/attn_bench.py                       # (2, 6), (16, 12), (64, 12)
    python tools/attn_bench.py --imgs 64 --heads 12  # one shape

Inputs are seeded, so the SHA-256 printed for each output identifies the result bytes across builds.  The card name,
its power limit and the SM clock read while the kernel runs are printed with the timings."""
import argparse
import hashlib
import os
import subprocess
import sys
import threading

import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mickey_b200 import _lib  # noqa: E402
from tests.gpu_util import stream  # noqa: E402


def smi(fields):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={fields}",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10)
        return r.stdout.strip() if r.returncode == 0 else "n/a"
    except (OSError, subprocess.TimeoutExpired):
        return "n/a"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--imgs", type=int, default=0)
    ap.add_argument("--heads", type=int, default=0)
    ap.add_argument("--T", type=int, default=1939)
    ap.add_argument("--iters", type=int, default=0, help="timed calls (default: 20, 10 at 64 images)")
    ap.add_argument("--impl", type=int, default=int(os.environ.get("ATTN_IMPL", "1")), help="1 wgmma, 2 mma.sync")
    a = ap.parse_args()
    shapes = [(a.imgs, a.heads)] if a.imgs else [(2, 6), (16, 12), (64, 12)]
    lib = _lib.load()
    T = a.T
    print(f"card: {torch.cuda.get_device_name()}  power limit: {smi('power.limit')} W  "
          f"max SM clock: {smi('clocks.max.sm')} MHz", flush=True)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for n_img, heads in shapes:
        D = heads * 64
        g = torch.Generator(device="cpu").manual_seed(1234 + n_img * 100 + heads)
        qkv = torch.randn(n_img * T, 3 * D, generator=g).half().cuda()
        att = torch.empty(n_img * T, D, dtype=torch.float16, device="cuda")
        fn = lambda: _lib.check(lib.mk_op_attention(_lib.ptr(qkv), _lib.ptr(att), n_img, T, D, heads, a.impl, stream()))
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        it = a.iters or (20 if n_img < 64 else 10)
        clocks = []
        stop = threading.Event()

        def sample():       # SM clock while the timed loop runs
            while not stop.is_set():
                c = smi("clocks.sm")
                if c.isdigit():
                    clocks.append(int(c))
                stop.wait(0.05)
        th = threading.Thread(target=sample)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        th.start()
        e0.record()
        for _ in range(it):
            fn()
        e1.record()
        torch.cuda.synchronize()
        stop.set()
        th.join()
        us = e0.elapsed_time(e1) / it * 1e3
        fl = n_img * heads * 4 * T * T * 64
        mhz = sorted(clocks)[len(clocks) // 2] if clocks else 0
        rate = f"{n_img * heads * T * T / us / n_sm / mhz:.2f} exp/clk/SM" if mhz else "exp rate n/a"
        sha = hashlib.sha256(att.cpu().numpy().tobytes()).hexdigest()[:16]
        print(f"impl={a.impl} imgs={n_img} heads={heads} T={T}: {us:9.1f} us  {fl / us / 1e6:7.1f} TFLOP/s  {rate} "
              f"(SM clock median {mhz} MHz over {len(clocks)} samples)  sha256 {sha}", flush=True)


if __name__ == "__main__":
    main()
