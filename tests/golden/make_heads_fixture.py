"""Record the train-mode forward and backward of the unmodified reference's four heads (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_heads_fixture.py

reference_heads_small.npz: lib/models/MicKey/modules/mickey_extractor.py::DeepResBlock_{det,offset,depth,desc}, imported
through oracle/ref_harness.py, built from cfg['MICKEY'] of tests/golden/reference_cfg_curriculum_learning.yaml with the
switch of each case changed (USE_SOFTMAX, USE_DEPTHSIGMOID, NORM_DSC on and off), run on the CPU in float32 as written,
in train mode, at B = 2, 15 x 14, with 1024 input channels.  Inputs, all from one torch.Generator seeded per case
(`case_inputs`, which tests/test_heads_host.py calls to rebuild them without the reference):
    weights of dim > 1   N(0, 1) / sqrt(fan_in), in named_parameters() order (trainable parameters only)
    norm weights         1 + 0.2 N(0, 1); norm biases 0.1 N(0, 1)
    running statistics   running_mean 0.1 N(0, 1), running_var 1 + 0.5 U(0, 1)
    x, g                 N(0, 1): the feature volume and the upstream gradient of the output
Keys "<case>/<name>" for name in out, every trainable parameter's gradient and every updated running statistic:
<name>/idx and <name>/val (a seeded sample of flat indices and the fp32 values there) and <name>/sum (the sum of all
values, in fp64); "<case>/checksum" is the fp64 sum of |x| + |g| + |every parameter|.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

FIXTURE = os.path.join(HERE, "reference_heads_small.npz")
B, H, W, CIN = 2, 15, 14, 1024
SAMPLES = 96
# case -> (head, config switch, value, seed)
CASES = {
    "det_softmax": ("det_head", ("KP_HEADS", "USE_SOFTMAX"), True, 300),
    "det_sigmoid": ("det_head", ("KP_HEADS", "USE_SOFTMAX"), False, 301),
    "offset": ("det_offset", None, None, 302),
    "depth_raw": ("depth_head", ("KP_HEADS", "USE_DEPTHSIGMOID"), False, 303),
    "depth_sigmoid": ("depth_head", ("KP_HEADS", "USE_DEPTHSIGMOID"), True, 304),
    "desc_norm": ("dsc_head", ("DSC_HEAD", "NORM_DSC"), True, 305),
    "desc_raw": ("dsc_head", ("DSC_HEAD", "NORM_DSC"), False, 306),
}
CLASSES = {"det_head": "DeepResBlock_det", "det_offset": "DeepResBlock_offset", "depth_head": "DeepResBlock_depth",
           "dsc_head": "DeepResBlock_desc"}


def case_config(case):
    from tests.golden.make_training_tree import training_cfg
    config = training_cfg()["MICKEY"]
    _, switch, value, _ = CASES[case]
    if switch is not None:
        config[switch[0]][switch[1]] = value
    return config


def case_inputs(module, seed):
    """Fill `module`'s trainable parameters and running statistics and draw x, g from one generator; returns (x, g)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if not p.requires_grad:
                continue
            if p.dim() > 1:
                p.copy_(torch.randn(p.shape, generator=g) / (p[0].numel() ** 0.5))
            elif name.endswith("weight"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
        for name, b in module.named_buffers():
            if name.endswith("running_mean"):
                b.copy_(0.1 * torch.randn(b.shape, generator=g))
            elif name.endswith("running_var"):
                b.copy_(1 + 0.5 * torch.rand(b.shape, generator=g))
        x = torch.randn(B, CIN, H, W, generator=g)
        k = {"det_offset": 2, "dsc_head": 128}.get(CASES_BY_SEED[seed], 1)
        gout = torch.randn(B, k, H, W, generator=g)
    return x, gout


CASES_BY_SEED = {seed: head for head, _, _, seed in CASES.values()}


def sample_idx(n, k, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(n, generator=g)[:min(k, n)].sort().values


def checksum(module, x, gout):
    return float(x.double().abs().sum() + gout.double().abs().sum() +
                 sum(p.detach().double().abs().sum() for p in module.parameters()))


def record(case, values, seed, out):
    for i, (name, v) in enumerate(values.items()):
        idx = sample_idx(v.numel(), SAMPLES, seed * 1000 + i)
        out[f"{case}/{name}/idx"] = idx.numpy().astype(np.int32)
        out[f"{case}/{name}/val"] = v.reshape(-1)[idx].numpy().astype(np.float32)
        out[f"{case}/{name}/sum"] = np.float64(v.double().sum())


def reference_module():
    from oracle import ref_harness
    assert ref_harness.available(), "reference tree not present (set MICKEY_REFERENCE_ROOT)"
    ref_harness._install_stubs()
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    try:
        with ref_harness._ref_on_path():
            import lib.models.MicKey.modules.mickey_extractor as mx
    finally:
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return mx


def main():
    mx = reference_module()
    out = {}
    for case, (head, _, _, seed) in CASES.items():
        torch.manual_seed(seed)
        m = getattr(mx, CLASSES[head])(case_config(case)).train()
        x, gout = case_inputs(m, seed)
        out[f"{case}/checksum"] = np.float64(checksum(m, x, gout))
        y = m(x)
        y.backward(gout)
        vals = {"out": y.detach()}
        vals.update({n: p.grad for n, p in m.named_parameters() if p.requires_grad})
        vals.update({n: b.clone() for n, b in m.named_buffers() if "running" in n})
        record(case, vals, seed, out)
    np.savez_compressed(FIXTURE, **out)
    print("wrote", FIXTURE, os.path.getsize(FIXTURE), "bytes")


if __name__ == "__main__":
    main()
