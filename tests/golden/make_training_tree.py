"""Record the parameter and buffer tree of the unmodified reference's MicKeyTrainingModel (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_training_tree.py

reference_training_tree.json: lib/models/MicKey/model.py::MicKeyTrainingModel(cfg) for the reference's
curriculum_learning.yaml (tests/golden/reference_cfg_curriculum_learning.yaml, DINOV2.FLOAT16: True), imported through
oracle/ref_harness.py's stubs with a synthetic ViT-L/14 in place of the downloaded DINOv2 weights.  Keys:
    "state":   [name, "param" | "buffer", shape, dtype, requires_grad] in model.state_dict() order
    "nonpersistent": the same for buffers outside the state dict
    "training": {module name: training flag} for every module
    "topK":    loss_fn.topK
"""
import json
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

TREE = os.path.join(HERE, "reference_training_tree.json")


def reference_training_model(cfg, variant="vitl"):
    """The reference's MicKeyTrainingModel(cfg) with a seeded synthetic DINOv2 of `variant` (vits / vitb / vitl)."""
    from oracle import ref_harness as rh
    assert rh.available(), "reference tree not present (set MICKEY_REFERENCE_ROOT)"
    rh._install_stubs()
    compat = os.path.join(ROOT, "compat")                # transforms3d, when the package is absent
    if compat not in sys.path:
        sys.path.append(compat)
    for name in ("matplotlib.pyplot", "matplotlib.cm"):
        sys.modules.setdefault(name, types.ModuleType(name))
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    orig_hub = torch.hub.load_state_dict_from_url
    try:
        with rh._ref_on_path():
            import lib.models.MicKey.modules.DINO_modules.dinov2 as dinov2
            import lib.models.MicKey.modules.mickey_extractor as mx
            from lib.models.MicKey.model import MicKeyTrainingModel
            factory = {"vits": dinov2.vit_small, "vitb": dinov2.vit_base, "vitl": dinov2.vit_large}[variant]
            mx.vit_large = factory
            torch.manual_seed(0)
            torch.hub.load_state_dict_from_url = lambda *a, **k: factory(
                img_size=518, patch_size=14, init_values=1.0, ffn_layer="mlp", block_chunks=0).state_dict()
            model = MicKeyTrainingModel(cfg)
    finally:
        torch.hub.load_state_dict_from_url = orig_hub
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return model


CONFIGS = ("curriculum_learning", "curriculum_learning_warm_up", "overlap_score", "overlap_score_warm_up")


def training_cfg(name="curriculum_learning"):
    """The reference's training config `name` (tests/golden/reference_cfg_<name>.yaml)."""
    from mickey_b200.config import default_cfg
    cfg = default_cfg()
    cfg.merge_from_file(os.path.join(HERE, f"reference_cfg_{name}.yaml"))
    return cfg


def tree_of(model):
    """The record this file writes, of any model."""
    params = dict(model.named_parameters())
    persistent = model.state_dict(keep_vars=True)
    entry = lambda n, t: [n, "param" if n in params else "buffer", list(t.shape), str(t.dtype).replace("torch.", ""),
                          bool(t.requires_grad)]
    return {"state": [entry(n, t) for n, t in persistent.items()],
            "nonpersistent": [entry(n, t) for n, t in model.named_buffers() if n not in persistent],
            "training": {n: m.training for n, m in model.named_modules()},
            "topK": getattr(model.loss_fn, "topK", None)}


def main():
    tree = tree_of(reference_training_model(training_cfg()))
    with open(TREE, "w") as f:
        json.dump(tree, f, indent=0)
    print("wrote", TREE, os.path.getsize(TREE), "bytes,", len(tree["state"]), "state entries")


if __name__ == "__main__":
    main()
