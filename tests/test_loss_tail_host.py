"""The CUDA loss tail's math and C ABI without a GPU.

- oracle.loss_tail_oracle.tail_closed_form (the arithmetic csrc/loss_tail.cu runs: the SVD-free rotation backward, the
  soft score's two paths, the VCRE / POSE_ERR and softmax backward) against fp64 autograd through the reference's helpers
  (tail_autograd: backproject_3d, weighted_procrustes with torch.svd, soft_inlier_counting_3d, compute_*_loss), to 1e-10
  of each gradient's largest magnitude, on every loss fixture with its recorded draws and on every combination of loss
  type, soft clipping and null hypothesis; the rotation backward alone on random H of both determinant signs.
- Each planted mutation of the closed form is rejected by the same comparison.
- mk_loss_tail_* reject every bad argument on the host, before anything is launched.
"""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.loss import LossParams
from oracle import loss_oracle as lo
from oracle import loss_tail_oracle as lto
from tests import loss_cases

FIX = np.load(loss_cases.FIXTURE)
REL = 1e-10


def _rel(got, want):
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-300))


def _problem(name, cfg=None):
    """fp64 CPU leaves, constants, the recorded draws and their inliers_final for fixture case `name`."""
    cfg = loss_cases.case_cfg(name) if cfg is None else cfg
    p = LossParams(cfg)
    batch = {k: v.double() for k, v in loss_cases.case_batch(name).items()}
    ref = lo.metric_pose_loss(batch, p, outer_idx=torch.from_numpy(FIX[f"{name}/outer_idx"]).long(),
                              inner_idx=torch.from_numpy(FIX[f"{name}/inner_idx"]).long())
    assert ref["num_valid_h"] == 1
    T = batch["T_0to1"]
    const = dict(K0=batch["K_color0"], K1=batch["K_color1"], Kori0=batch["Kori_color0"], Kori1=batch["Kori_color1"],
                 Rgt=T[:, :3, :3].clone(), tgt=T[:, :3, 3:].transpose(1, 2).clone(), sampled=ref["sampled"],
                 inl=ref["inliers_final"])
    leaves = [batch[k].clone().requires_grad_() for k in ("kps0", "depth_kp0", "kps1", "depth_kp1")]
    return p, leaves, const


def _upstream(p, B, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B * p.it_matches, generator=g, dtype=torch.float64) for _ in range(3)]


def _autograd(p, leaves, const, ups):
    out = lto.tail_autograd(*leaves, const["K0"], const["K1"], const["Kori0"], const["Kori1"], const["Rgt"], const["tgt"],
                            const["sampled"], const["inl"], p)
    assert out is not None
    grads = torch.autograd.grad(sum((o * u).sum() for o, u in zip(out, ups)), leaves)
    return [o.detach() for o in out], grads


def _closed(p, leaves, const, ups, mutation=None):
    return lto.tail_closed_form(*leaves, const["K0"], const["K1"], const["Kori0"], const["Kori1"], const["Rgt"],
                                const["tgt"], const["sampled"], const["inl"], p, *ups, mutation=mutation)


def _worst(p, leaves, const, ups, mutation=None):
    """max over the values and the four gradients of |closed form - autograd| / max |autograd|."""
    vals, grads = _autograd(p, leaves, const, ups)
    cf = _closed(p, leaves, const, ups, mutation)
    errs = [_rel(cf[k], v) for k, v in zip(("loss_value", "loss_rot", "loss_trans"), vals)]
    errs += [_rel(cf[k], g) for k, g in zip(("dkps0", "ddepth0", "dkps1", "ddepth1"), grads)]
    return max(errs)


@pytest.mark.parametrize("name", list(loss_cases.CASES))
def test_closed_form_matches_autograd_on_fixture_cases(name):
    p, leaves, const = _problem(name)
    err = _worst(p, leaves, const, _upstream(p, leaves[0].shape[0], 1))
    assert err <= REL, err


LOSS_VARIANTS = list(itertools.product(("VCRE", "POSE_ERR"), (True, False), (True, False)))


@pytest.mark.parametrize("loss,soft,null", LOSS_VARIANTS)
def test_closed_form_matches_autograd_on_every_loss_variant(loss, soft, null):
    p, leaves, const = _problem("vits_vcre", loss_cases.loss_cfg(loss, soft, null))
    err = _worst(p, leaves, const, _upstream(p, leaves[0].shape[0], 2))
    assert err <= REL, err


def _random_H(n, seed):
    g = torch.Generator().manual_seed(seed)
    H = torch.randn(n, 3, 3, generator=g, dtype=torch.float64)
    want = torch.ones(n, dtype=torch.float64)
    want[n // 2:] = -1                                                   # first half det > 0, second half det < 0
    H[:, 0] *= (torch.sign(torch.linalg.det(H)) * want).unsqueeze(-1)
    return H, torch.randn(n, 3, 3, generator=g, dtype=torch.float64)


def _svd_rotation(H):
    """weighted_procrustes's R = V Z U^T from H, in autograd through torch.svd."""
    U, _, V = torch.svd(H)
    Z = torch.eye(3, dtype=H.dtype).repeat(H.shape[0], 1, 1)
    Z[:, -1, -1] = torch.sign(torch.linalg.det(U @ V.transpose(1, 2)))
    return V @ Z @ U.transpose(1, 2)


def test_rotation_backward_matches_svd_autograd_on_random_H():
    H, G = _random_H(4000, 5)
    dets = torch.linalg.det(H)
    assert int((dets < 0).sum()) == 2000 and int((dets > 0).sum()) == 2000
    Hl = H.clone().requires_grad_()
    R = _svd_rotation(Hl)
    (want,) = torch.autograd.grad((R * G).sum(), Hl)
    got = lto.procrustes_backward(R.detach(), H, G)
    err = ((got - want).abs().amax((1, 2)) / want.abs().amax((1, 2))).max()
    assert float(err) <= REL, float(err)
    for mutation in ("rt_sign", "z_in_m"):
        bad = lto.procrustes_backward(R.detach(), H, G, mutation)
        assert float(((bad - want).abs().amax((1, 2)) / want.abs().amax((1, 2))).max()) > 1e-3, mutation


@pytest.mark.parametrize("mutation", ["rt_sign", "score_direct", "mean_x"])
def test_mutations_are_rejected_on_the_fixture(mutation):
    p, leaves, const = _problem("vits_vcre")
    ups = _upstream(p, leaves[0].shape[0], 3)
    assert _worst(p, leaves, const, ups) <= REL
    assert _worst(p, leaves, const, ups, mutation) > 1e-4


def test_acos_clip_edge_mutation_is_rejected():
    """A hypothesis whose rotation equals the ground truth has cos = 1, clipped: autograd passes no gradient there."""
    p, leaves, const = _problem("vits_pose")
    ups = _upstream(p, leaves[0].shape[0], 4)
    R = _closed(p, leaves, const, ups)["R"]
    const["Rgt"][0] = R[0]
    assert _worst(p, leaves, const, ups) <= REL
    assert _worst(p, leaves, const, ups, "acos_edge") > 1e-4


# ---- the C ABI's host checks ------------------------------------------------------------------------------------------
GOOD = dict(B=2, N=1938, IM=20, IR=20, S=512, loss_type=0, th=0.15, temp=0.05)
FAKE = C.c_void_p(0x10000)


def _forward(lib, null=None, ws_bytes=None, null_hyp=1, null_score=10.0, **kw):
    a = dict(GOOD, **kw)
    ptrs = [FAKE] * 17                # 12 inputs, 3 outputs, status, workspace
    if null is not None:
        ptrs[null] = None
    ws = lib.mk_loss_tail_ws_bytes(GOOD["B"], GOOD["N"], GOOD["IM"], GOOD["IR"], GOOD["S"]) if ws_bytes is None else ws_bytes
    return lib.mk_loss_tail_forward(*ptrs[:12], a["B"], a["N"], a["IM"], a["IR"], a["S"], a["loss_type"], 1, null_hyp,
                                    a["th"], a["temp"], null_score, 0.9, *ptrs[12:], ws, None)


def _backward(lib, null=None, ws_bytes=None, **kw):
    a = dict(GOOD, **kw)
    ptrs = [FAKE] * 20                # 12 inputs, 3 upstream gradients, 4 outputs, workspace
    if null is not None:
        ptrs[null] = None
    ws = lib.mk_loss_tail_ws_bytes(GOOD["B"], GOOD["N"], GOOD["IM"], GOOD["IR"], GOOD["S"]) if ws_bytes is None else ws_bytes
    return lib.mk_loss_tail_backward(*ptrs[:12], a["B"], a["N"], a["IM"], a["IR"], a["S"], a["loss_type"], 1, 1, a["th"],
                                     a["temp"], *ptrs[12:], ws, None)


BAD_SIZES = [dict(B=0), dict(B=65536), dict(N=0), dict(N=46341), dict(IM=0), dict(IR=0), dict(IR=-3), dict(S=0),
             dict(S=48), dict(S=2080), dict(S=16), dict(B=65535, IM=200, IR=200), dict(loss_type=2), dict(loss_type=-1),
             dict(th=0.0), dict(th=float("nan")), dict(th=float("inf")), dict(temp=0.0), dict(temp=float("nan"))]


def _ids(kw):
    return ",".join(f"{k}={v}" for k, v in kw.items())


@pytest.mark.parametrize("kw", BAD_SIZES + [dict(null=i) for i in range(17)] + [dict(ws_bytes=1000)] +
                         [dict(null_score=float("inf")), dict(null_score=float("nan"))], ids=_ids)
def test_forward_rejects_bad_arguments_before_launching(kw):
    """MK_ERR_INVALID with a message from the host checks: nothing is launched (without a GPU a launch would return
    MK_ERR_CUDA instead)."""
    lib = _lib.load()
    assert _forward(lib, **kw) == -1
    assert b"mk_loss_tail_forward" in lib.mk_last_error()


@pytest.mark.parametrize("kw", BAD_SIZES + [dict(null=i) for i in range(20)] + [dict(ws_bytes=1000)], ids=_ids)
def test_backward_rejects_bad_arguments_before_launching(kw):
    lib = _lib.load()
    assert _backward(lib, **kw) == -1
    assert b"mk_loss_tail_backward" in lib.mk_last_error()


def test_workspace_size_rejects_unsupported_sizes():
    lib = _lib.load()
    assert lib.mk_loss_tail_ws_bytes(8, 1938, 20, 20, 512) > 0
    for args in ((0, 1938, 20, 20, 512), (8, 1938, 20, 20, 500), (8, 1938, 0, 20, 512), (8, 1938, 20, 0, 512)):
        assert lib.mk_loss_tail_ws_bytes(*args) == -1


# ---- use_cuda_modules(model, cuda_tail=True) ------------------------------------------------------------------------
def test_use_cuda_modules_sets_the_tail_flag_on_the_recorded_tree():
    from mickey_b200.loss import MetricPoseLoss
    from mickey_b200.training import use_cuda_modules
    from tests.test_heads_host import model_from_tree
    model = use_cuda_modules(model_from_tree())
    loss = model.loss_fn
    assert type(loss) is MetricPoseLoss and loss.cuda_tail is False          # the default keeps the autograd tail
    assert use_cuda_modules(model, cuda_tail=True) is model
    assert model.loss_fn is loss and loss.cuda_tail is True                  # the drop-in already there gets the flag
    use_cuda_modules(model)                                                  # a second call changes nothing
    use_cuda_modules(model, cuda_tail=True)
    assert model.loss_fn is loss and loss.cuda_tail is True
    fresh = use_cuda_modules(model_from_tree(), cuda_tail=True)
    assert type(fresh.loss_fn) is MetricPoseLoss and fresh.loss_fn.cuda_tail is True
