"""The heads' transformer without a GPU: the drop-in's parameter tree and PE buffer against the live reference class,
the fp64 restatement against fp64 autograd of the oracle, the bounds against an fp32 restatement and the planted
mutations, and every rejection of the Python surface."""
import os

import numpy as np
import pytest
import torch

from mickey_b200.head_transformer import Transformer_self_att, head_transformer
from oracle import mickey_oracle as mo
from oracle import ref_harness
from tests import head_transformer_check as hc

SD_KEYS = {"q_proj": "q_proj.weight", "k_proj": "k_proj.weight", "v_proj": "v_proj.weight", "merge": "merge.weight",
           "mlp0": "mlp.0.weight", "mlp2": "mlp.2.weight", "norm1_w": "norm1.weight", "norm1_b": "norm1.bias",
           "norm2_w": "norm2.weight", "norm2_b": "norm2.bias"}


def _reference_class():
    if not ref_harness.available():
        pytest.skip("reference tree not present")
    import sys
    ref_harness._install_stubs()
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    try:
        with ref_harness._ref_on_path():
            from lib.models.MicKey.modules.att_layers.transformer import Transformer_self_att as Ref
    finally:
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return Ref


@pytest.mark.parametrize("layers", [1, 3])
@pytest.mark.parametrize("pe_on", [False, True])
def test_parameter_tree_matches_reference(layers, pe_on):
    Ref = _reference_class()
    ref, ours = Ref(128, layers, pe_on), Transformer_self_att(128, layers, pe_on)
    rs, os_ = ref.state_dict(), ours.state_dict()
    assert list(rs) == list(os_)
    assert all(rs[k].shape == os_[k].shape for k in rs)
    assert [n for n, _ in ref.named_buffers()] == [n for n, _ in ours.named_buffers()] == ["posEnc.pe"]
    assert torch.equal(ref.posEnc.pe, ours.posEnc.pe)
    assert (ours.d_model, ours.nheads, ours.layer_names, ours.add_posEnc) == \
        (ref.d_model, ref.nheads, ref.layer_names, ref.add_posEnc)
    ours.load_state_dict(rs, strict=True)
    ref.load_state_dict(os_, strict=True)


def test_constructor_rejections():
    with pytest.raises(ValueError):
        Transformer_self_att(256, 3)
    with pytest.raises(ValueError):
        Transformer_self_att(128, 0)
    with pytest.raises(ValueError):
        Transformer_self_att(128, 1025)


@pytest.mark.parametrize("B,h,w,L,pe_on", [(2, 15, 14, 3, True), (3, 7, 9, 1, False), (2, 1, 33, 3, True)])
def test_restatement_equals_fp64_autograd_and_bounds_hold(B, h, w, L, pe_on):
    x, params, go = hc.case_inputs(B, h, w, L, seed=B + h + w)
    pe = Transformer_self_att(128, L, pe_on).posEnc.pe if pe_on else None
    ref = hc.restate(x, params, pe, go)
    xd = x.double().requires_grad_()
    pd = [p.double().requires_grad_() for p in params]
    sd = {f"att.layers.{i // 10}.{SD_KEYS[hc.NAMES[i % 10]]}": p for i, p in enumerate(pd)}
    out = mo.head_transformer(sd, "att.", xd, pe_on)
    grads = torch.autograd.grad(out, [xd] + pd, go.double())
    scale = lambda t: float(t.abs().max()) + 1e-300
    assert float((out.detach() - ref["out"][0]).abs().max()) <= 1e-12 * scale(out)
    assert float((grads[0] - ref["dx"][0]).abs().max()) <= 1e-12 * scale(grads[0])
    for i, g in enumerate(grads[1:]):
        assert float((g - ref[hc.param_key(i)][0]).abs().max()) <= 1e-12 * scale(g), hc.param_key(i)
    r32 = hc.restate(x, params, pe, go, dtype=torch.float32)
    for k, (v, _) in r32.items():
        hc.check(k, v, *ref[k])
    for mut in hc.MUTATIONS:
        if mut == "pe_next" and not pe_on:
            continue
        assert hc.rejected(ref, hc.restate(x, params, pe, go, mutation=mut)), mut


def _params(L=3, device="cpu"):
    return [p for l in Transformer_self_att(128, L).to(device).layers for p in l.params()]


@pytest.mark.parametrize("make", [
    lambda: (torch.zeros(1, 128, 4, 4, dtype=torch.float64), {}),                 # dtype
    lambda: (torch.zeros(1, 128, 4, 4), {}),                                      # CPU device
    lambda: (torch.zeros(1, 64, 4, 4), {}),                                       # C != 128
    lambda: (torch.zeros(0, 128, 4, 4), {}),                                      # B = 0
    lambda: (torch.zeros(128, 4, 4), {}),                                         # not 4-D
    lambda: (torch.zeros(1, 128, 257, 4), {"pe": True}),                          # h > 256 with the PE
    lambda: (torch.zeros(1, 128, 4, 257), {"pe": True}),                          # w > 256 with the PE
    lambda: (torch.zeros(1, 128, 4, 4), {"params_device": "meta"}),               # parameters elsewhere
    lambda: ("not a tensor", {}),
    lambda: (torch.zeros(1, 128, 1, 1).expand(65536, 128, 1, 1), {}),                             # B above the grid limit
    lambda: (torch.zeros(1, 128, 1, 1).expand(1, 128, 2048, 2049), {}),                           # tokens above the grid limit
])
def test_rejections(make):
    x, kw = make()
    params = _params(device=kw.get("params_device", "cpu"))
    pe = Transformer_self_att(128, 1, True).posEnc.pe if kw.get("pe") else None
    with pytest.raises(ValueError):
        head_transformer(x, params, pe)


def test_module_rejects_input_elsewhere():
    m = Transformer_self_att(128, 3, True)
    with pytest.raises(ValueError):
        m(torch.zeros(2, 128, 300, 4))
    with pytest.raises(ValueError):
        m(torch.zeros(2, 128, 5, 4))          # CPU input: the kernels run on CUDA only


def _fixture_module():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_head_transformer_fixture.py")
    spec = importlib.util.spec_from_file_location("make_head_transformer_fixture", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


REF_TO_KEY = {f"layers.{i}.{v}": f"L{i}.{k}" for i in range(3) for k, v in SD_KEYS.items()}


@pytest.mark.parametrize("case", ["pe", "nope"])
def test_golden_reference_within_bounds_of_fp64(case):
    """The unmodified reference's fp32 forward and backward (tests/golden/reference_head_transformer_small.npz) lie within
    the fp32 bounds of the fp64 restatement and of fp64 autograd of the oracle, at every recorded element and in every
    tensor's sum."""
    fx = _fixture_module()
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_head_transformer_small.npz"))
    pe_on, seed = fx.CASES[case]
    m = Transformer_self_att(128, fx.LAYERS, pe_on)
    x, gout = fx.case_inputs(m, seed)
    assert fx.checksum(m, x, gout) == float(z[f"{case}/checksum"]), "the seeded inputs are no longer reproduced"
    params = [p.detach() for layer in m.layers for p in layer.params()]
    ref = hc.restate(x, params, m.posEnc.pe if pe_on else None, gout)
    xd = x.double().requires_grad_()
    pd = [p.double().requires_grad_() for p in params]
    sd = {f"att.layers.{i // 10}.{SD_KEYS[hc.NAMES[i % 10]]}": p for i, p in enumerate(pd)}
    out = mo.head_transformer(sd, "att.", xd, pe_on)
    grads = torch.autograd.grad(out, [xd] + pd, gout.double())
    oracle = {"out": out.detach(), "dx": grads[0]}
    oracle.update({hc.param_key(i): g for i, g in enumerate(grads[1:])})
    names = ["out", "dx"] + list(REF_TO_KEY)
    for name in names:
        key = REF_TO_KEY.get(name, name)
        value, bound = ref[key]
        idx = torch.from_numpy(z[f"{case}/{name}/idx"].astype(np.int64))
        got = torch.from_numpy(z[f"{case}/{name}/val"]).double()
        for want in (value, oracle[key]):
            err = (got - want.reshape(-1)[idx]).abs()
            assert bool((err <= bound.reshape(-1)[idx]).all()), (case, name, float((err / bound.reshape(-1)[idx]).max()))
            assert abs(float(z[f"{case}/{name}/sum"]) - float(want.sum())) <= float(bound.sum()), (case, name)
