"""Device times of the ViT-B GEMMs at the C3 batch (64 images = 124096 tokens) and of the head convolution, for A/B runs of
GEMM changes:   python tools/gemm_bench.py [n_images] [impl ...]

impl: "tc" (the default dispatch), "paired" / "unpaired" (the persistent kernel with / without two-CTA pairs sharing
B).  Several impls are timed in the same process, alternating, three rounds each.

Next to each ViT GEMM's rate it prints the HBM bytes of two traffic models and the bandwidth they imply at the measured
time.  "m-fastest" is a tile order that walks the M-tiles fastest: A (far larger than the L2) is evicted before the grid
reaches the next column of N-tiles, so it is read once per column.  "n-fastest" is gemm_tile()'s order: every A
row-panel is read once while all of B stays in L2.  Both count B once, the output once and the fp32 residual of RESID_F
twice (read and write).  The bytes are computed from the shapes, not measured."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mickey_b200 import _lib  # noqa: E402
from tests.gpu_util import IMPL, gemm  # noqa: E402

IMPL.update(paired=3, unpaired=4)
lib = _lib.load()
dev = "cuda"
n_img = int(sys.argv[1]) if len(sys.argv) > 1 else 64
impls = sys.argv[2:] or ["tc"]
ROUNDS = 3 if len(impls) > 1 else 1
M, D = n_img * 1939, 768
tag = torch.cuda.get_device_name(0)
torch.manual_seed(0)


def timeit1(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def timeit(fn):
    """{impl: [us per call of each round]} with fn(impl) run for every impl in turn, ROUNDS times."""
    res = {i: [] for i in impls}
    for _ in range(ROUNDS):
        for i in impls:
            res[i].append(timeit1(lambda: fn(i)))
    return res


def show(res):
    return "  ".join(f"{i} " + "/".join(f"{u:.1f}" for u in us) + " us" for i, us in res.items())


def lin(N_, K_, epi, **kw):
    a = torch.randn(M, K_, device=dev).half()
    w = (torch.randn(N_, K_, device=dev) * 0.02).half()
    return lambda impl: gemm(epi, a, w, M, N_, K_, impl=impl, **kw)


x32 = torch.randn(M, D, device=dev)
g = torch.randn(D, device=dev) * 0.1
total = {i: 0.0 for i in impls}
for name, N_, K_, epi, kw in (
        ("qkv", 3 * D, D, "STORE_H", dict(bias=torch.randn(3 * D, device=dev), out_h=torch.empty(M, 3 * D, dtype=torch.float16, device=dev), out_h_ld=3 * D)),
        ("proj", D, D, "RESID_F", dict(bias=torch.randn(D, device=dev), gamma=g, out_f=x32, out_f_ld=D)),
        ("fc1+gelu", 4 * D, D, "STORE_H", dict(bias=torch.randn(4 * D, device=dev), act=1, out_h=torch.empty(M, 4 * D, dtype=torch.float16, device=dev), out_h_ld=4 * D)),
        ("fc2", D, 4 * D, "RESID_F", dict(bias=torch.randn(D, device=dev), gamma=g, out_f=x32, out_f_ld=D))):
    res = timeit(lin(N_, K_, epi, **kw))
    for i in impls:
        total[i] += min(res[i])
    us = min(res[impls[0]])
    a_bytes, rest = M * K_ * 2, N_ * K_ * 2 + (M * N_ * 2 if epi == "STORE_H" else 2 * M * N_ * 4)
    traffic = {"m-fastest": a_bytes * (N_ // 128) + rest, "n-fastest": a_bytes + rest}
    model = "  ".join(f"{k} {b / 1e9:5.2f} GB = {b / us / 1e3:5.0f} GB/s" for k, b in traffic.items())
    print(f"{tag} vit-b.{name:9s} {M}x{N_}x{K_}: {show(res)}  {impls[0]}: {2 * M * N_ * K_ / us / 1e6:7.1f} TFLOP/s  {model}",
          flush=True)
    del kw
print(f"{tag} vit-b block GEMMs (sum of the fastest rounds): " + "  ".join(f"{i} {t:.1f} us" for i, t in total.items()), flush=True)
big = 16384
obig = torch.empty(big, 4096, dtype=torch.float16, device=dev)
a = torch.randn(big, 4096, device=dev).half(); w = (torch.randn(4096, 4096, device=dev) * 0.02).half()
res = timeit(lambda impl: gemm("STORE_H", a, w, big, 4096, 4096, impl=impl, out_h=obig, out_h_ld=4096))
us = min(res[impls[0]])
print(f"{tag} gemm 16384x4096x4096: {show(res)}  {impls[0]}: {2 * big * 4096 * 4096 / us / 1e6:7.1f} TFLOP/s", flush=True)
h2, w2, G, Cc = 53, 40, 4, 512
R = n_img * h2 * w2
a = torch.randn(R, G * Cc, device=dev).half()
w = (torch.randn(G * Cc, 9 * Cc, device=dev) * 0.01).half()
bb = torch.randn(G * Cc, device=dev)
out = torch.empty(R, G * Cc, dtype=torch.float16, device=dev)
taps = [(ky - 1) * w2 + (kx - 1) for ky in range(3) for kx in range(3)]
res = timeit(lambda impl: gemm("CONV", a, w, R, Cc, impl=impl, taps=taps, chunks_per_tap=Cc // 64, groups=G, a_col_group_off=Cc,
                               b_row_group_off=Cc, bias=bb, bias_group_off=Cc, act=2, pad_h2=h2, pad_w2=w2, out_h=out,
                               out_h_ld=G * Cc, out_h_group_off=Cc))
us = min(res[impls[0]])
print(f"{tag} head.conv3x3 4x(512->512), {n_img} images: {show(res)}  {impls[0]}: {2 * R * G * Cc * 9 * Cc / us / 1e6:7.1f} TFLOP/s",
      flush=True)
