"""Record the forward and backward of the unmodified reference's BasicBlock (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_resblock_fixture.py

reference_resblock_small.npz: lib/models/MicKey/modules/utils/extractor_utils.py::BasicBlock(cin, cout), imported through
oracle/ref_harness.py, run on the CPU in float32 as written, in train mode, at B = 2 and 15 x 14, for the five block shapes
of the heads with relu True and False.  Inputs, all from one torch.Generator seeded per case (`case_inputs`, which
tests/test_resblock_host.py calls to rebuild them without the reference):
    convs    N(0, 1) / sqrt(fan_in), in named_parameters() order
    bn       weight 1 + 0.2 N(0, 1), bias 0.1 N(0, 1); running_mean 0.1 N(0, 1), running_var 1 + 0.5 U(0, 1)
    x, g     N(0, 1): the input and the upstream gradient of the output
Keys "<case>/<name>" for name in out, dx, every parameter gradient and the four updated running statistics
("bn1.running_mean", ...): <name>/idx and <name>/val (a seeded sample of flat indices and the fp32 values there) and
<name>/sum (the sum of all values, in fp64); "<case>/checksum" is the fp64 sum of |x| + |g| + |every parameter|.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

FIXTURE = os.path.join(HERE, "reference_resblock_small.npz")
B, H, W = 2, 15, 14
SHAPES = [(1024, 512), (512, 256), (256, 128), (128, 64), (128, 128)]
CASES = {f"{ci}_{co}_{'relu' if r else 'norelu'}": (ci, co, r, 100 + 2 * i + (0 if r else 1))
         for i, (ci, co) in enumerate(SHAPES) for r in (True, False)}
SAMPLES = 256


def case_inputs(module, seed):
    """Fill `module`'s parameters and running statistics and draw x, g from one generator; returns (x, g)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
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
    cin, cout = module.conv1.in_channels, module.conv1.out_channels
    x = torch.randn(B, cin, H, W, generator=g)
    gout = torch.randn(B, cout, H, W, generator=g)
    return x, gout


def sample_idx(n, k, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(n, generator=g)[:min(k, n)].sort().values


def checksum(module, x, gout):
    return float(x.double().abs().sum() + gout.double().abs().sum() +
                 sum(p.detach().double().abs().sum() for p in module.parameters()))


def reference_class():
    from oracle import ref_harness
    assert ref_harness.available(), "reference tree not present (set MICKEY_REFERENCE_ROOT)"
    ref_harness._install_stubs()
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    try:
        with ref_harness._ref_on_path():
            from lib.models.MicKey.modules.utils.extractor_utils import BasicBlock
    finally:
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return BasicBlock


def main():
    Ref = reference_class()
    out = {}
    for case, (ci, co, relu, seed) in CASES.items():
        m = Ref(ci, co).train()
        x, gout = case_inputs(m, seed)
        out[f"{case}/checksum"] = np.float64(checksum(m, x, gout))
        xx = x.clone().requires_grad_()
        y = m(xx, relu=relu)
        y.backward(gout)
        vals = {"out": y.detach(), "dx": xx.grad}
        vals.update({n: p.grad for n, p in m.named_parameters()})
        vals.update({n: b.clone() for n, b in m.named_buffers() if "running" in n})
        for i, (name, v) in enumerate(vals.items()):
            idx = sample_idx(v.numel(), SAMPLES, seed * 1000 + i)
            out[f"{case}/{name}/idx"] = idx.numpy().astype(np.int32)
            out[f"{case}/{name}/val"] = v.reshape(-1)[idx].numpy().astype(np.float32)
            out[f"{case}/{name}/sum"] = np.float64(v.double().sum())
    np.savez_compressed(FIXTURE, **out)
    print("wrote", FIXTURE, os.path.getsize(FIXTURE), "bytes")


if __name__ == "__main__":
    main()
