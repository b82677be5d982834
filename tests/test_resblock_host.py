"""The residual block without a GPU: the drop-in's parameter tree against the live reference class, strict state-dict
loads, the oracle's closed-form backward against fp64 autograd, its running-statistics update against F.batch_norm, and
every rejection of the Python surface and of the workspace-size functions."""
import sys

import pytest
import torch
import torch.nn as nn

from mickey_b200 import _lib
from mickey_b200.resblock import BasicBlock
from oracle import ref_harness
from oracle import resblock_oracle as ro

SHAPES = [(1024, 512), (512, 256), (256, 128), (128, 64), (128, 128)]


def _reference_class():
    if not ref_harness.available():
        pytest.skip("reference tree not present")
    ref_harness._install_stubs()
    saved = {k: v for k, v in sys.modules.items() if k == "lib" or k.startswith("lib.")}
    for k in saved:
        del sys.modules[k]
    try:
        with ref_harness._ref_on_path():
            from lib.models.MicKey.modules.utils.extractor_utils import BasicBlock as Ref
    finally:
        for k in [k for k in sys.modules if k == "lib" or k.startswith("lib.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return Ref


@pytest.mark.parametrize("cin,cout", SHAPES)
@pytest.mark.parametrize("bn", [True, False])
def test_parameter_tree_matches_reference(cin, cout, bn):
    Ref = _reference_class()
    torch.manual_seed(0)
    ref = Ref(cin, cout, bn=bn)
    torch.manual_seed(0)
    ours = BasicBlock(cin, cout, bn=bn)
    sr, so = ref.state_dict(), ours.state_dict()
    assert list(sr) == list(so)
    for k in sr:
        assert sr[k].shape == so[k].shape and sr[k].dtype == so[k].dtype
        assert torch.equal(sr[k], so[k]), k            # same construction order: same initial values
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in ours.named_parameters()]
    assert [type(m).__name__ for m in ref.modules()][1:] == [type(m).__name__ for m in ours.modules()][1:]
    ours.load_state_dict(sr, strict=True)
    ref.load_state_dict(so, strict=True)


def _rand_block(cin, cout, bn, seed):
    torch.manual_seed(seed)
    m = BasicBlock(cin, cout, bn=bn).double()
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-0.2, 0.2)
                mod.running_mean.uniform_(-0.1, 0.1)
                mod.running_var.uniform_(0.5, 2.0)
    return m


@pytest.mark.parametrize("cin,cout", [(64, 32), (32, 32)])
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("bn", [True, False])
def test_closed_form_backward_equals_fp64_autograd(cin, cout, train, relu, bn):
    m = _rand_block(cin, cout, bn, 3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, cin, 5, 6, generator=g, dtype=torch.float64, requires_grad=True)
    go = torch.randn(2, cout, 5, 6, generator=g, dtype=torch.float64)
    ps = dict(w1=m.conv1.weight.detach().clone().requires_grad_(), w2=m.conv2.weight.detach().clone().requires_grad_(),
              wsc=m.shortcut[0].weight.detach().clone().requires_grad_() if cin != cout else None)
    bn1, bn2 = ro.bn_params(m.bn1), ro.bn_params(m.bn2)
    for b in (bn1, bn2):
        if b is not None:
            b["weight"].requires_grad_()
            b["bias"].requires_grad_()
    out, aux = ro.block_forward(x, ps["w1"], ps["w2"], ps["wsc"], bn1, bn2, train, relu)
    out.backward(go)
    with torch.no_grad():
        cf = ro.block_backward(x, ps["w1"], ps["w2"], ps["wsc"], bn1, bn2, go, aux, train, relu)
    auto = dict(dx=x.grad, w1=ps["w1"].grad, w2=ps["w2"].grad, wsc=None if ps["wsc"] is None else ps["wsc"].grad,
                bn1_w=None if bn1 is None else bn1["weight"].grad, bn1_b=None if bn1 is None else bn1["bias"].grad,
                bn2_w=None if bn2 is None else bn2["weight"].grad, bn2_b=None if bn2 is None else bn2["bias"].grad)
    for k, v in auto.items():
        if v is None:
            assert cf[k] is None, k
            continue
        assert ((cf[k] - v).norm() / v.norm()).item() <= 1e-12, k


def test_oracle_matches_module_forward_and_running_statistics():
    m = _rand_block(64, 32, True, 5)
    x = torch.randn(3, 64, 4, 7, dtype=torch.float64)
    w1, w2, wsc = m.conv1.weight.detach(), m.conv2.weight.detach(), m.shortcut[0].weight.detach()
    bn1, bn2 = ro.bn_params(m.bn1), ro.bn_params(m.bn2)
    out, aux = ro.block_forward(x, w1, w2, wsc, bn1, bn2, True, True)
    # the same block through torch modules in train mode
    F = torch.nn.functional
    with torch.no_grad():
        a1 = F.relu(m.bn1(m.conv1(x)))
        ref = F.relu(m.bn2(m.conv2(a1)) + m.shortcut(x))
    assert ((out - ref).abs().max() / ref.abs().max()).item() < 1e-12
    for b, mod, mean, var in ((bn1, m.bn1, aux["mean1"], aux["var1"]), (bn2, m.bn2, aux["mean2"], aux["var2"])):
        rm, rv = ro.running_update(b, mean, var, 3 * 4 * 7)
        assert torch.allclose(rm, mod.running_mean, rtol=1e-12, atol=1e-15)
        assert torch.allclose(rv, mod.running_var, rtol=1e-12, atol=1e-15)
        # planted: the biased variance in running_var is rejected
        biased = (1 - b["factor"]) * b["running_var"] + b["factor"] * var
        assert not torch.allclose(biased, mod.running_var, rtol=1e-6, atol=0)


def test_constructor_rejections():
    with pytest.raises(ValueError, match="stride"):
        BasicBlock(64, 64, stride=2)
    with pytest.raises(ValueError, match="padding_mode"):
        BasicBlock(64, 64, padding_mode="reflect")
    for cin, cout in ((48, 64), (64, 40), (16, 16), (8192, 64)):
        with pytest.raises(ValueError, match="multiple of 32"):
            BasicBlock(cin, cout)


def test_forward_rejections_before_any_launch():
    m = BasicBlock(64, 32)
    with pytest.raises(ValueError, match="float32"):
        m(torch.zeros(1, 64, 4, 4, dtype=torch.float64))
    with pytest.raises(ValueError, match="float32"):
        m(torch.zeros(1, 32, 4, 4))
    with pytest.raises(ValueError, match="B, h, w"):
        m(torch.zeros(0, 64, 4, 4))
    with pytest.raises(ValueError, match="at most"):
        m(torch.zeros(1, 64, 4100, 4100, device="meta"))
    with pytest.raises(ValueError, match="more than 1 value"):
        m(torch.zeros(1, 64, 1, 1))
    with pytest.raises(ValueError, match="CUDA"):
        m(torch.zeros(1, 64, 2, 2))
    m.eval()
    with pytest.raises(ValueError, match="CUDA"):          # B h w = 1 is fine in eval mode
        m(torch.zeros(1, 64, 1, 1))
    m.train()
    m.bn1.eval()
    with pytest.raises(ValueError, match="both"):
        m(torch.zeros(1, 64, 2, 2))
    m3 = BasicBlock(64, 32)
    m3.bn2 = nn.Identity()
    with pytest.raises(ValueError, match="BatchNorm2d or both nn.Identity"):
        m3(torch.zeros(1, 64, 2, 2, device="meta"))
    assert int(m3.bn1.num_batches_tracked) == 0
    for kw in (dict(affine=False), dict(track_running_stats=False)):
        m2 = BasicBlock(64, 32)
        m2.bn2 = nn.BatchNorm2d(32, **kw)
        with pytest.raises(ValueError, match="affine"):
            m2(torch.zeros(1, 64, 2, 2))


def test_workspace_sizes_reject_bad_geometries():
    lib = _lib.load()
    assert lib.mk_resblock_ws_bytes(2, 15, 14, 128, 64) > 0
    assert lib.mk_resblock_backward_ws_bytes(2, 15, 14, 128, 64) > 0
    assert lib.mk_resblock_saved_bytes(2, 15, 14, 128, 64) > 0
    bad = [(0, 4, 4, 64, 64), (1, 0, 4, 64, 64), (1, 4, 0, 64, 64), (1, 4, 4, 48, 64), (1, 4, 4, 64, 16),
           (1, 4, 4, 8192, 64), (1, 4096, 4096, 64, 64), (-1, 4, 4, 64, 64)]
    for args in bad:
        assert lib.mk_resblock_ws_bytes(*args) == -1, args
        assert lib.mk_resblock_saved_bytes(*args) == -1, args
        assert lib.mk_resblock_backward_ws_bytes(*args) == -1, args
    assert lib.mk_op_conv_tf32_ws_bytes(0, 1, 4, 4, 64, 64, 9) > 0
    for args in ((3, 1, 4, 4, 64, 64, 9), (0, 1, 4, 4, 64, 64, 4), (2, 1, 4, 4, 40, 64, 9)):
        assert lib.mk_op_conv_tf32_ws_bytes(*args) == -1, args


def test_c_entry_points_reject_bad_arguments():
    """Host checks return MK_ERR_INVALID with a message before touching any pointer (the pointers here are bogus)."""
    import ctypes as C
    lib = _lib.load()
    P = _lib.MkResblockParams()
    st = (C.c_longlong * 4)(0, 0, 0, 0)
    fake = C.c_void_p(256)
    rc = lib.mk_resblock_forward(fake, st, 1, 4, 4, 64, 64, C.byref(P), 0, fake, fake, 1 << 30, fake, 1 << 30, None)
    assert rc == -1 and b"w1" in lib.mk_last_error()
    P.w1 = P.w2 = 256
    rc = lib.mk_resblock_forward(fake, st, 1, 4, 4, 64, 48, C.byref(P), 0, fake, fake, 1 << 30, fake, 1 << 30, None)
    assert rc == -1
    rc = lib.mk_resblock_forward(fake, st, 1, 1, 1, 64, 64, C.byref(P), 1 | 8, fake, fake, 1 << 30, fake, 1 << 30, None)
    assert rc == -1                                           # BN without its parameters
    rc = lib.mk_resblock_forward(fake, st, 1, 4, 4, 64, 64, C.byref(P), 0, fake, fake, 1 << 30, fake, 16, None)
    assert rc == -1 and b"workspace" in lib.mk_last_error()
    G = _lib.MkResblockGrads()
    rc = lib.mk_resblock_backward(fake, fake, st, fake, 1, 4, 4, 64, 64, C.byref(P), 2, 1, C.byref(G), fake, 1 << 30, None)
    assert rc == -1 and b"dx" in lib.mk_last_error()
    G.wsc = 256
    rc = lib.mk_resblock_backward(fake, fake, st, fake, 1, 4, 4, 64, 64, C.byref(P), 2, 8, C.byref(G), fake, 1 << 30, None)
    assert rc == -1 and b"no such parameter" in lib.mk_last_error()
    rc = lib.mk_op_conv_tf32(0, fake, fake, fake, 1, 4, 4, 64, 64, 9, fake, 16, None)
    assert rc == -1


def test_reference_fixture_reproduced_by_the_oracle():
    """The unmodified reference block's fp32 CPU run (tests/golden/reference_resblock_small.npz) against the oracle in
    fp64 on inputs rebuilt without the reference: sampled values within fp32 rounding of the fp64 result (relative to
    the quantity's scale; gradients, where fp32 flips a few ReLU masks, within 3 % in norm), full sums to 1e-5 (1e-3 for
    gradients) of their absolute sums, and
    the planted biased running variance rejected."""
    import numpy as np
    from tests.golden import make_resblock_fixture as fx
    data = np.load(fx.FIXTURE)
    for case, (ci, co, relu, seed) in fx.CASES.items():
        m = BasicBlock(ci, co)
        x, gout = fx.case_inputs(m, seed)
        assert abs(fx.checksum(m, x, gout) - float(data[f"{case}/checksum"])) <= 1e-9 * float(data[f"{case}/checksum"])
        m = m.double()
        w1, w2 = m.conv1.weight.detach(), m.conv2.weight.detach()
        wsc = m.shortcut[0].weight.detach() if hasattr(m, "shortcut") else None
        bn1, bn2 = ro.bn_params(m.bn1), ro.bn_params(m.bn2)
        out, aux = ro.block_forward(x.double(), w1, w2, wsc, bn1, bn2, True, relu)
        gr = ro.block_backward(x.double(), w1, w2, wsc, bn1, bn2, gout.double(), aux, True, relu)
        M = 2 * 15 * 14
        rm1, rv1 = ro.running_update(bn1, aux["mean1"], aux["var1"], M)
        rm2, rv2 = ro.running_update(bn2, aux["mean2"], aux["var2"], M)
        ref = {"out": out, "dx": gr["dx"], "conv1.weight": gr["w1"], "conv2.weight": gr["w2"],
               "bn1.weight": gr["bn1_w"], "bn1.bias": gr["bn1_b"], "bn2.weight": gr["bn2_w"], "bn2.bias": gr["bn2_b"],
               "bn1.running_mean": rm1, "bn1.running_var": rv1, "bn2.running_mean": rm2, "bn2.running_var": rv2}
        if wsc is not None:
            ref["shortcut.0.weight"] = gr["wsc"]
        for name, r in ref.items():
            flat = r.reshape(-1)
            idx = torch.from_numpy(data[f"{case}/{name}/idx"].astype(np.int64))
            val = torch.from_numpy(data[f"{case}/{name}/val"]).double()
            if "running" in name or name == "out":        # element-wise, within fp32 rounding of the scale
                err = (val - flat[idx]).abs().max().item() / flat.abs().max().item()
                assert err <= 1e-5, (case, name, err)
            else:                                         # gradients: fp32 flips some ReLU masks, so a relative norm
                err = ((val - flat[idx]).norm() / flat[idx].norm()).item()
                assert err <= 3e-2, (case, name, err)
            s = float(data[f"{case}/{name}/sum"])
            stol = 1e-5 if "running" in name or name == "out" else 1e-3
            assert abs(s - flat.sum().item()) <= stol * flat.abs().sum().item(), (case, name)
        biased = (1 - bn1["factor"]) * bn1["running_var"] + bn1["factor"] * aux["var1"]
        idx = torch.from_numpy(data[f"{case}/bn1.running_var/idx"].astype(np.int64))
        val = torch.from_numpy(data[f"{case}/bn1.running_var/val"]).double()
        assert (val - biased[idx]).abs().max().item() > 1e-5 * rv1.abs().max().item()
