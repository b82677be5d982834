"""Record the forward and backward of the unmodified reference's Transformer_self_att (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_head_transformer_fixture.py

reference_head_transformer_small.npz: lib/models/MicKey/modules/att_layers/transformer.py::Transformer_self_att(128, 3,
add_posEnc), imported through oracle/ref_harness.py, run on the CPU in float32 as written, at B = 2 and 15 x 14, with the
positional encoding on ("pe") and off ("nope").  Inputs, all from one torch.Generator seeded with SEED per case
(`case_inputs`, which tests/test_head_transformer_host.py calls to rebuild them without the reference):
    weights  nn.init.xavier_uniform_ over the module's matrices in parameters() order (the reference's own init, seeded)
    norms    gamma = 1 + 0.2 N(0, 1), beta = 0.1 N(0, 1), perturbed away from 1 and 0
    x, g     N(0, 1) [2, 128, 15, 14]: the input and the upstream gradient of the output
Keys "<case>/<name>" for name in out, dx and the 30 parameter gradients ("layers.<i>.<param>"):
    <name>/idx, <name>/val   a seeded sample of flat indices and the reference's fp32 values there (the file stays small)
    <name>/sum               the sum of all its fp32 values, in fp64
and "<case>/checksum": the sum of |x| + |g| + |every parameter| in fp64, which the test compares to catch a generator
that no longer reproduces the inputs.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

FIXTURE = os.path.join(HERE, "reference_head_transformer_small.npz")
B, H, W, LAYERS = 2, 15, 14, 3
CASES = {"pe": (True, 11), "nope": (False, 12)}          # case -> (add_posEnc, seed)
SAMPLES_OUT, SAMPLES_PARAM = 2048, 256


def case_inputs(module, seed):
    """Fill `module`'s parameters (in parameters() order) and draw x, g from one generator; returns (x, g)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if p.dim() > 1:
                torch.nn.init.xavier_uniform_(p, generator=g)
            elif name.endswith("weight"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    x = torch.randn(B, 128, H, W, generator=g)
    gout = torch.randn(B, 128, H, W, generator=g)
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
            from lib.models.MicKey.modules.att_layers.transformer import Transformer_self_att
    finally:
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return Transformer_self_att


def main():
    Ref = reference_class()
    out = {}
    for case, (pe_on, seed) in CASES.items():
        m = Ref(128, LAYERS, pe_on)
        x, gout = case_inputs(m, seed)
        xx = x.clone().requires_grad_()
        y = m(xx)
        y.backward(gout)
        vals = {"out": y.detach(), "dx": xx.grad}
        vals.update({n: p.grad for n, p in m.named_parameters()})
        for i, (name, v) in enumerate(vals.items()):
            k = SAMPLES_OUT if name in ("out", "dx") else SAMPLES_PARAM
            idx = sample_idx(v.numel(), k, seed * 1000 + i)
            out[f"{case}/{name}/idx"] = idx.numpy().astype(np.int32)
            out[f"{case}/{name}/val"] = v.reshape(-1)[idx].numpy().astype(np.float32)
            out[f"{case}/{name}/sum"] = np.float64(v.double().sum())
        out[f"{case}/checksum"] = np.float64(checksum(m, x, gout))
    np.savez_compressed(FIXTURE, **out)
    print("wrote", FIXTURE, os.path.getsize(FIXTURE), "bytes")


if __name__ == "__main__":
    main()
