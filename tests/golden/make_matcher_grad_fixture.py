"""Record autograd through the matcher of the unmodified reference (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_matcher_grad_fixture.py

reference_matcher_grad_small.npz: the reference's dualSoftmax module (lib/models/MicKey/modules/utils/feature_matcher.py),
ComputeCorrespondences.kp_matrix_scores (compute_correspondences.py:46-50) and `final_scores = scores * kp_scores`
(model.py:201), on the golden features of the ViT-S / ViT-B small cases, TEMPERATURE 0.1, on the CPU in float32 as written.
For every case of CASES, keys "<case>/<name>", on the first pair of the loss case's batch (B = 1; every pair is computed
independently, so one pair per case keeps the file small without losing a code path):
    ddsc0, ddsc1 [1, 128, N], dscr0, dscr1 [1, 1, N]   the gradients of the module's inputs
    ddustbin (scalar; dustbin cases only)             dustbin_score.grad
Upstream gradients:
    "reinforce": torch.autograd.backward(torch.log(final + 1e-16), probs_grad) (model.py:118-134) with the recorded
                 REINFORCE probs_grad of reference_loss_small.npz (case vits_vcre / vitb_vcre);
    "dense":     torch.autograd.backward((scores, kp_scores), (Gs, Gk)) with Gs, Gk = dense_grads(B, N, seed).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402

FIXTURE = os.path.join(HERE, "reference_matcher_grad_small.npz")
TEMPERATURE = 0.1
# case -> (golden features, loss case whose first pair (and its probs_grad) is used, upstream, USE_DUSTBIN): each features
# set, each upstream and each dustbin setting once
CASES = {
    "vits_reinforce_dust": ("vits_small", "vits_vcre", "reinforce", True),
    "vitb_dense_nodust": ("vitb_small", "vitb_vcre", "dense", False),
}
LOSS_PAIRS = {"vits_vcre": [0, 1], "vitb_vcre": [0, 0]}      # tests/loss_cases.py CASES


def dense_grads(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, N, N, generator=g), torch.randn(B, N, N, generator=g)


def inputs(feat, loss):
    """(dsc0, dsc1, scr0, scr1, probs_grad) of the case: the first pair the loss fixture took from the golden features."""
    z = np.load(os.path.join(HERE, f"{feat}.npz"))
    take = lambda k: torch.from_numpy(z[k][LOSS_PAIRS[loss]]).float()
    d0, d1, s0, s1 = take("dsc0"), take("dsc1"), take("scr0"), take("scr1")
    B, N = d0.shape[0], d0.shape[2]
    r = np.load(os.path.join(HERE, "reference_loss_small.npz"))
    pg = torch.zeros(B * N * N)
    pg[torch.from_numpy(r[f"{loss}/grad_idx"]).long()] = torch.from_numpy(r[f"{loss}/grad_val"])
    return d0[:1], d1[:1], s0[:1], s1[:1], pg.reshape(B, N, N)[:1]


def reference_modules():
    assert ref_harness.available(), "reference tree not present"
    ref_harness._install_stubs()
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    with ref_harness._ref_on_path():
        import lib.models.MicKey.modules.utils.feature_matcher as fm
        import lib.models.MicKey.modules.compute_correspondences as cc
    for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    return fm, cc


def record():
    fm, cc = reference_modules()
    out = {}
    for i, (name, (feat, loss, up, dust)) in enumerate(CASES.items()):
        d0, d1, s0, s1, pg = inputs(feat, loss)
        d0.requires_grad_(); d1.requires_grad_(); s0.requires_grad_(); s1.requires_grad_()
        m = fm.dualSoftmax({"TEMPERATURE": TEMPERATURE, "USE_DUSTBIN": dust})
        scores = m(d0, d1)
        kp = cc.ComputeCorrespondences.kp_matrix_scores(None, s0, s1)
        final = scores * kp
        if up == "reinforce":
            torch.autograd.backward(torch.log(final + 1e-16), pg)
        else:
            B, N = scores.shape[0], scores.shape[1]
            torch.autograd.backward((scores, kp), dense_grads(B, N, 100 + i))
        p = f"{name}/"
        out.update({p + "ddsc0": d0.grad.numpy(), p + "ddsc1": d1.grad.numpy(), p + "dscr0": s0.grad.numpy(),
                    p + "dscr1": s1.grad.numpy()})
        if dust:
            out[p + "ddustbin"] = np.float32(m.dustbin_score.grad.item())
        print(f"{name}: |ddsc0| {d0.grad.norm():.4e} |dscr0| {s0.grad.norm():.4e}", flush=True)
    return out


def seed_of(name):
    return 100 + list(CASES).index(name)


if __name__ == "__main__":
    rec = record()
    np.savez_compressed(FIXTURE, **rec)
    print("wrote", FIXTURE, os.path.getsize(FIXTURE), "bytes")
