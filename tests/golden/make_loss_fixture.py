"""Record MetricPoseLoss (lib/models/MicKey/modules/loss/loss_class.py) of the unmodified reference (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_loss_fixture.py

  reference_loss_small.npz, for every case of tests/loss_cases.py CASES (the ViT-S / ViT-B small golden features with a
  planted geometry; VCRE and POSE_ERR, soft clipping on and off, null hypothesis on and off, top-K at B = 4), keys
  "<case>/<name>":
    outer_idx int32 [B*IM, S], inner_idx int32 [B*IM*IR, C]   both torch.multinomial draws (:138, :159), recorded by
                                                              wrapping the call
    avg_loss, baseline [B], loss_value [B*IM]                 the REINFORCE baseline and each outer iteration's loss
    scores [B*IM*IR], inliers_final uint8 [B*IM*IR, S/8]      soft score and final inlier mask (np.packbits, little bit
                                                              order) of every hypothesis
    grad_idx int64 [M], grad_val float32 [M]                  the nonzero entries of gradients[0] (flat [B*N*N] index)
    kps0_grad, kps1_grad, depth0_grad, depth1_grad            after avg_loss.backward()
    num_valid_h, mask_topk, avg_loss_rot, avg_loss_trans
  "vcre_grid" float64 [196, 3]: the reference's eye_coords_glob[:, :3] (lib/benchmarks/reprojection.py:32-60).

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_loss_fixture.py --warm-up

  reference_loss_warmup_small.npz, the same keys for every case of tests/loss_cases.py WARMUP_CASES: the reference's two
  warm-up configs (64 samples per set, no null hypothesis; top-K at B = 4 in the curriculum one), VCRE and POSE_ERR.
The reference runs on the CPU in float32, as written.
"""
import contextlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402
from tests import loss_cases  # noqa: E402


def reference_loss_module():
    """Import loss_class from the reference tree, with stubs for its plotting / quaternion imports."""
    assert ref_harness.available(), "reference tree not present"
    ref_harness._install_stubs()
    if "transforms3d" not in sys.modules:
        t3 = types.ModuleType("transforms3d")
        t3.quaternions = types.ModuleType("transforms3d.quaternions")
        t3.quaternions.quat2mat = None            # unused by the loss
        sys.modules["transforms3d"], sys.modules["transforms3d.quaternions"] = t3, t3.quaternions
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    with ref_harness._ref_on_path():
        import lib.models.MicKey.modules.loss.loss_class as lc
        import lib.benchmarks.reprojection as rp
    for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    return lc, rp


@contextlib.contextmanager
def recording(lc):
    """Record both torch.multinomial draws, every weighted_procrustes mask, the soft scores and the locals of
    single_iteration_RANSAC at its return."""
    rec = {"draws": [], "w": [], "scores": [], "locals": None}
    mult, wp, sc = torch.multinomial, lc.weighted_procrustes, lc.soft_inlier_counting_3d

    def multinomial(*a, **k):
        r = mult(*a, **k)
        rec["draws"].append(r.clone())
        return r

    def procrustes(*a, **k):
        rec["w"].append(k.get("w"))
        return wp(*a, **k)

    def scores(*a, **k):
        r = sc(*a, **k)
        rec["scores"].append(r.detach().clone())
        return r

    def prof(frame, event, arg):
        if event == "return" and frame.f_code.co_name == "single_iteration_RANSAC":
            rec["locals"] = dict(frame.f_locals)

    torch.multinomial, lc.weighted_procrustes, lc.soft_inlier_counting_3d = multinomial, procrustes, scores
    sys.setprofile(prof)
    try:
        yield rec
    finally:
        sys.setprofile(None)
        torch.multinomial, lc.weighted_procrustes, lc.soft_inlier_counting_3d = mult, wp, sc


def record(cases=loss_cases.CASES, seed0=1000):
    lc, rp = reference_loss_module()
    out = {"vcre_grid": np.asarray(rp.eye_coords_glob[:, :3], dtype=np.float64)}
    for i, name in enumerate(cases):
        torch.manual_seed(seed0 + i)
        batch = loss_cases.case_batch(name)
        loss = lc.MetricPoseLoss(loss_cases.case_cfg(name))
        with recording(lc) as rec:
            avg_loss, outputs, grads, num_valid_h = loss(batch)
        avg_loss.backward()
        loc = rec["locals"]
        assert num_valid_h == 1 and len(rec["draws"]) == 2, (name, num_valid_h, len(rec["draws"]))
        B = batch["final_scores"].shape[0]
        g = grads[0].detach().reshape(-1)
        nz = torch.nonzero(g).reshape(-1)
        inl = rec["w"][-1].detach().numpy().astype(np.uint8)
        p = f"{name}/"
        out.update({
            p + "outer_idx": rec["draws"][0].numpy().astype(np.int32),
            p + "inner_idx": rec["draws"][1].numpy().astype(np.int32),
            p + "avg_loss": np.float32(avg_loss.item()),
            p + "baseline": (loc["baseline"].detach() / loss.it_matches).numpy(),
            p + "loss_value": loc["loss_value"].detach().reshape(-1).numpy(),
            p + "scores": rec["scores"][-1].reshape(-1).numpy(),
            p + "inliers_final": np.packbits(inl, axis=1, bitorder="little"),
            p + "grad_idx": nz.numpy(), p + "grad_val": g[nz].numpy(),
            p + "num_valid_h": np.int32(num_valid_h),
            p + "mask_topk": outputs["mask_topk"].numpy(),
            p + "avg_loss_rot": np.float32(outputs["avg_loss_rot"].item()),
            p + "avg_loss_trans": np.float32(outputs["avg_loss_trans"].item()),
        })
        for k in ("kps0", "kps1", "depth0", "depth1"):
            out[p + k + "_grad"] = outputs[k].grad.numpy()
        n_inl = inl.reshape(-1, inl.shape[-1]).sum(1)
        print(f"{name}: B {B} avg_loss {avg_loss.item():.6f} grad nnz {nz.numel()} final inliers min/mean/max "
              f"{n_inl.min()}/{n_inl.mean():.1f}/{n_inl.max()}", flush=True)
    return out


if __name__ == "__main__":
    if "--warm-up" in sys.argv[1:]:
        path, rec = loss_cases.WARMUP_FIXTURE, record(loss_cases.WARMUP_CASES, 2000)
    else:
        path, rec = loss_cases.FIXTURE, record()
    np.savez_compressed(path, **rec)
    print("wrote", path, os.path.getsize(path), "bytes")
