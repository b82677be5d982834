"""Record featureMatcher.get_matches_list (feature_matcher.py:19-46) of the unmodified reference (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_matches_fixture.py

  reference_matches_720x540.npz  for the 720x540 ViT-S and ViT-B golden cases (tests/common.py GOLDEN_CASES), every pair b,
                                 both matrices (final_scores, scores) and four min_conf values:
                                   "<case>/<matrix>/<b>/min_conf"     float64 [4]: 0, 1 (drops the all-zero rows) and exp() of
                                                                      the median and 90th percentile of the min_conf = 0 scores
                                   "<case>/<matrix>/<b>/<k>/matches"  int16 [M, 2], the reference's output for min_conf[k]
                                   "<case>/<matrix>/<b>/scores"       float64 [N-1], the row maxima of scores[b, :-1, :-1]
                                 (the score of a match (i, j) is the maximum of row i; equal scores form the tied blocks whose
                                 order the reference's unstable sort leaves open)

The reference model is evaluated in float64 (as make_reference_fixtures.stagewise does), so the matrices the test rebuilds
with the oracle agree with the reference's to ~1e-15 and the argmaxes do not depend on the CPU.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402

CASES = ("vits_720x540", "vitb_720x540")


def record():
    from mickey_b200.config import mickey_cfg
    from mickey_b200.weights import synthetic_state_dict
    from tests.common import GOLDEN_CASES, float64_eval, synthetic_pair, to_float64
    out = {}
    for name in CASES:
        spec = GOLDEN_CASES[name]
        cfg = mickey_cfg(spec["variant"], spec["it_matches"], spec["it_ransac"], float16=False)
        sd = synthetic_state_dict(cfg, seed=spec["weight_seed"])
        model = ref_harness.build_reference_model(cfg, sd, variant=spec["variant"]).double()
        for m in model.modules():
            if hasattr(m, "amp_dtype"):
                m.amp_dtype = torch.float64
        data = to_float64(synthetic_pair(spec["batch"], spec["height"], spec["width"], seed=spec["data_seed"]))
        with torch.no_grad(), float64_eval():
            model.compute_matches(data)
            data["final_scores"] = data["scores"] * data["kp_scores"]           # compute_pose.py:23
            matcher = model.compute_matches.matcher
            for mat in ("final_scores", "scores"):
                for b in range(spec["batch"]):
                    s = data[mat][b:b + 1]
                    out[f"{name}/{mat}/{b}/scores"] = s[0, :-1, :-1].max(1).values.numpy()
                    m0 = matcher.get_matches_list(s, 0.0)
                    kept = s[0, m0[:, 0], m0[:, 1]]
                    q = torch.quantile(kept, torch.tensor([0.5, 0.9], dtype=kept.dtype))
                    confs = [0.0, 1.0] + [float(torch.exp(v)) for v in q]
                    out[f"{name}/{mat}/{b}/min_conf"] = np.array(confs)
                    for k, c in enumerate(confs):
                        out[f"{name}/{mat}/{b}/{k}/matches"] = matcher.get_matches_list(s, c).numpy().astype(np.int16)
        print(name, "done", flush=True)
    return out


if __name__ == "__main__":
    assert ref_harness.available(), "set MICKEY_REFERENCE_ROOT to a reference checkout"
    np.savez_compressed(os.path.join(HERE, "reference_matches_720x540.npz"), **record())
