"""Time one MicKey training step on a model moved onto the CUDA modules by mickey_b200.training.use_cuda_modules.

    python tools/train_step_bench.py [--rounds 3] [--steps 5] [--warmup 2] [--out result.json]

The step is the reference's training_step (model.py:51-59, backward_step :91-147) on seeded synthetic weights and images,
ViT-L with the fp16 backbone: two extractor calls, the matcher, kp_scores and final_scores, one MetricPoseLoss call,
avg_loss.backward(), backward_step's torch.autograd.backward, clip_grad_norm_(max_norm=5) and Adam (lr 1e-4, eps 1e-6).
Two configurations: B = 8 at 720x540 (curriculum_learning) and B = 24 at 480x360 (curriculum_learning_warm_up).

Each is run two ways, alternated round by round after every shape is warmed up:
    cuda   the heads are the CUDA drop-ins (mickey_b200.heads)
    eager  the heads are oracle/heads_oracle.py's head_chain in eager fp32 torch (default TF32 flags) on the same
           Parameters; backbone, matcher and loss are the CUDA modules in both
CUDA events split the step into: backbone (both calls), each head's forward (both calls), matcher + kp_scores, loss
(forward and avg_loss.backward), the backward through heads and matcher, and clip + Adam.  The backward is not split by
head: autograd runs the heads' backward interleaved.  Peak memory is torch.cuda.max_memory_allocated over a step.  The
card's name and power limit are read in the same run.  Needs a CUDA device; there is no CPU fallback.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import heads_oracle as ho  # noqa: E402
from tests.test_gpu_heads_training import converted_model, correspondences, match, step_batch  # noqa: E402

CONFIGS = {"b8_720x540": ("curriculum_learning", 8, 720, 540), "b24_480x360": ("curriculum_learning_warm_up", 24, 480, 360)}
HEADS = ("det_offset", "depth_head", "det_head", "dsc_head")


def eager_heads(model):
    """Each head as head_chain over the CUDA head's own Parameters and buffers (gradients land in the same .grad)."""
    ex = model.compute_matches.extractor
    config = model.cfg["MICKEY"]
    fns = {}
    for n in HEADS:
        sd = dict(getattr(ex, n).state_dict(keep_vars=True))
        fns[n] = (lambda f, sd=sd, n=n: ho.head_chain(sd, n, config, f)[0])
    return fns


def one_step(model, opt, ims, data, heads, ev):
    ex = model.compute_matches.extractor
    mark = lambda k: ev.setdefault(k, torch.cuda.Event(enable_timing=True)).record()
    opt.zero_grad(set_to_none=True)
    mark("start")
    feats = []
    for i, im in enumerate(ims):
        f, _ = extract_backbone(ex, im)
        feats.append(f)
    mark("backbone")
    cs = []
    outs = [{}, {}]
    for n in HEADS:
        for i, f in enumerate(feats):
            outs[i][n] = heads[n](f)
        mark(f"head {n}")
    for i in range(2):
        cs.append(correspondences(*(outs[i][n] for n in HEADS)))
    final = match(model.compute_matches.matcher.matching_mat, cs[0], cs[1])
    mark("matcher")
    batch = dict(data, final_scores=final, kps0=cs[0][0], kps1=cs[1][0], depth_kp0=cs[0][1], depth_kp1=cs[1][1])
    avg_loss, outputs, probs_grad, num_its = model.loss_fn(batch)
    avg_loss.backward()
    mark("loss")
    up = (probs_grad[0], outputs["kps0"].grad, outputs["kps1"].grad, outputs["depth0"].grad, outputs["depth1"].grad)
    torch.autograd.backward((torch.log(final + 1e-16), cs[0][0], cs[1][0], cs[0][1], cs[1][1]), up)
    mark("backward")
    torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=5)
    opt.step()
    mark("optimiser")


def extract_backbone(ex, im):
    B, _, H, W = im.shape
    f = 14
    im = im[:, :, :f * (H // f), :f * (W // f)]
    with torch.no_grad():
        feats = ex.dinov2_vitl14.forward_features(im.to(torch.float16))["x_norm_patchtokens"].permute(0, 2, 1).reshape(
            B, 1024, H // f, W // f).float()
    return feats, None


def split(ev):
    keys = list(ev)
    out = {}
    for a, b in zip(keys, keys[1:]):
        out[b] = ev[a].elapsed_time(ev[b])
    out["step"] = ev[keys[0]].elapsed_time(ev[keys[-1]])
    return out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_step_bench needs a CUDA device")
    result = {"card": card(), "configs": {}}
    for cname, (config, B, H, W) in CONFIGS.items():
        torch.manual_seed(0)
        model = converted_model(config)
        opt = torch.optim.Adam(model.parameters(), lr=1e-4, eps=1e-6)
        ims, data = step_batch(B, H, W, seed=B)
        ex = model.compute_matches.extractor
        variants = {"cuda": {n: getattr(ex, n) for n in HEADS}, "eager": eager_heads(model)}
        for heads in variants.values():
            for _ in range(a.warmup):
                one_step(model, opt, ims, data, heads, {})
        torch.cuda.synchronize()
        times = {v: [] for v in variants}
        peaks = {}
        for _ in range(a.rounds):
            for v, heads in variants.items():
                torch.cuda.reset_peak_memory_stats()
                for _ in range(a.steps):
                    ev = {}
                    one_step(model, opt, ims, data, heads, ev)
                    torch.cuda.synchronize()
                    times[v].append(split(ev))
                peaks[v] = max(peaks.get(v, 0), torch.cuda.max_memory_allocated())
        result["configs"][cname] = {
            v: {"median_ms": {k: statistics.median(t[k] for t in times[v]) for k in times[v][0]},
                "min_step_ms": min(t["step"] for t in times[v]), "max_step_ms": max(t["step"] for t in times[v]),
                "peak_mb": peaks[v] / 2 ** 20, "steps": len(times[v])} for v in variants}
        del model, opt
        torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
