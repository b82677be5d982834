"""Map-free steps with the reference image extracted once (feature banks) against the paired path.

    python tools/shared_reference_bench.py                        # ViT-B, 1024 hypotheses, 32 pairs of 720x540
    python tools/shared_reference_bench.py --variant vits --it-matches 8 --it-ransac 64

Every pair of a step shares one reference image, as every val/test pair of a Map-free scene does.  Seeded synthetic
images and weights.  Timed with CUDA events after warm-up, each mode in its own window:
  (a) model.forward on the explicit pairs: 2B images extracted per step; eager (like for like with (b), (c)) and replayed
      from CUDA graphs (the default forward)
  (b) extract_features on the B + 1 distinct images, then pose_from_features
  (c) the steady state of a scene: the reference's features cached, extract_features on the B queries, pose_from_features
It also reports the gather kernel's time (CUDA events around its launches), checks that (b) and (c) give the pose of (a)
under the same torch seed, and prints the card's name and power limit read in the same run.  One JSON line on stdout.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info(torch):
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        info["power_limit"] = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        info["power_limit"] = None
    return info


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--variant", default="vitb", choices=["vits", "vitb", "vitl"])
    ap.add_argument("--it-matches", type=int, default=16)
    ap.add_argument("--it-ransac", type=int, default=64)
    ap.add_argument("--pairs", type=int, default=32, help="queries per step, all against one reference")
    ap.add_argument("--height", type=int, default=720)
    ap.add_argument("--width", type=int, default=540)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch
    os.environ.setdefault("MICKEY_SYNTHETIC_BACKBONE", "1")
    from mickey_b200.config import mickey_cfg
    from mickey_b200.model import MickeyRelativePose
    from mickey_b200.weights import synthetic_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("shared_reference_bench.py measures on a CUDA device (an H100); none is available")

    dev = torch.device("cuda", 0)
    cfg = mickey_cfg(args.variant, args.it_matches, args.it_ransac)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=args.seed), strict=True)
    model = model.to(dev).eval()
    B, H, W = args.pairs, args.height, args.width
    g = torch.Generator().manual_seed(args.seed + 1)
    ref = torch.rand(1, 3, H, W, generator=g).to(dev)
    queries = torch.rand(B, 3, H, W, generator=g).to(dev)
    K = torch.tensor([[549.7, 0.0, 268.7], [0.0, 549.7, 351.8], [0.0, 0.0, 1.0]], device=dev)[None].repeat(B, 1, 1)
    pairs = {"image0": ref.expand(B, -1, -1, -1).contiguous(), "image1": queries, "K_color0": K, "K_color1": K}
    distinct = torch.cat([ref, queries])
    ref_idx, query_idx = [0] * B, list(range(B))

    def run_a(graphs):
        def step():
            model.use_graph = graphs
            d = dict(pairs)
            model(d)
            return d
        return step

    def run_b():
        f = model.extract_features(distinct)
        return model.pose_from_features(f, ref_idx, f, [i + 1 for i in query_idx], K, K)

    ref_feats = model.extract_features(ref)

    def run_c():
        return model.pose_from_features(ref_feats, ref_idx, model.extract_features(queries), query_idx, K, K)

    def timed(step, warmup=args.warmup):
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        return {"ms_per_step": round(ms, 3), "pairs_per_s": round(B / ms * 1e3, 2)}

    res = {"variant": args.variant, "hypotheses": args.it_matches * args.it_ransac, "pairs": B, "image": [H, W]}
    res.update(card_info(torch))
    res["a_forward_eager"] = timed(run_a(False))
    res["a_forward_graphs"] = timed(run_a(True), max(args.warmup, 4))     # both buffer sets captured before timing
    res["b_extract_all_then_pairs"] = timed(run_b)
    res["c_reference_cached"] = timed(run_c)

    # same seed, same pose: the banks reproduce the paired path bit for bit
    torch.manual_seed(123)
    a = run_a(False)()
    torch.manual_seed(123)
    b = run_b()
    torch.manual_seed(123)
    c = run_c()
    res["bitwise_equal_pose"] = {"b": all(torch.equal(a[k], b[k]) for k in ("R", "t", "inliers")),
                                 "c": all(torch.equal(a[k], c[k]) for k in ("R", "t", "inliers"))}

    # the gather kernel alone: CUDA events around each of its launches, over the same steps as (c)
    eng = model._engine()
    eng.profile(True)
    for _ in range(args.iters):
        run_c()
    prof = eng.profile_read()
    eng.profile(False)
    n, ms = prof.get("pairs.gather", (0, 0.0))
    res["gather_ms_per_step"] = round(ms / max(n, 1), 4)
    res["stage_ms_per_step_c"] = {k: round(v[1] / args.iters, 3) for k, v in prof.items()}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
