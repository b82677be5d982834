"""The dual-softmax matcher's forward on caller descriptors and its CUDA backward (csrc/matcher_grad.cu), element by
element against the fp64 closed form, with the bounds derived in tests/matcher_grad_check.py.

A failure names the output, the pair, the row or column, the channel and the 64-wide tile of the worst element.
"""
import time

import pytest
import torch

from mickey_b200.dual_softmax import dual_softmax, dualSoftmax
from oracle import mickey_oracle as mo
from tests import loss_cases
from tests import matcher_grad_check as mgc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
RATIOS = {}

# (B, N, T, dustbin, gradients, scale, pitch): scale None = unit descriptors, else Gaussian * scale (wide logits)
CASES = (
    [(3 if N <= 257 else 1, N, 0.1, True, "skf", None, None) for N in (2, 127, 128, 129, 255, 257, 850, 1938, 2303, 4176)]
    + [(8, 1938, 0.1, True, "skf", None, 1952), (24, 850, 0.1, True, "skf", None, 864),       # the two training shapes
       (24, 850, 0.1, False, "f", None, None)]
    + [(3, 257, 0.1, d, g, None, None) for d in (True, False) for g in ("s", "k", "f", "skf")]
    + [(2, 300, T, True, "skf", None, None) for T in (0.01, 1.0)] + [(2, 300, 0.01, False, "f", None, 320)]
    + [(2, 500, 0.1, True, "skf", 1.0, None), (2, 500, 0.01, False, "skf", 0.3, None)]
)


def _ids(c):
    B, N, T, d, g, sc, p = c
    return f"B{B}-N{N}-T{T}-{'dust' if d else 'nodust'}-{g}" + (f"-x{sc}" if sc else "") + (f"-p{p}" if p else "")


def run(args, scr=True):
    """(outputs of the forward, gradients of the inputs) of dual_softmax with the given upstream gradients."""
    d0, d1, T, dust, s0, s1, gs, gk, gf = args
    leaves = [None if t is None else t.clone().requires_grad_() for t in (d0, d1, dust, s0, s1)]
    x0, x1, a, y0, y1 = leaves
    out = dual_softmax(x0, x1, a, T, y0, y1) if scr else (dual_softmax(x0, x1, a, T),)
    ups = [(o, g) for o, g in zip(out, (gs, gk, gf)) if g is not None]
    torch.autograd.backward([o for o, _ in ups], [g for _, g in ups])
    grads = {k: None if t is None else t.grad for k, t in zip(("ddsc0", "ddsc1", "ddustbin", "dscr0", "dscr1"), leaves)}
    return out, grads


def compare(label, args, grads, fw=None, bw=None):
    d0, d1, T, dust, s0, s1, gs, gk, gf = args
    if fw is None:
        fw, bw = mgc.reference(*args)
    bnd = mgc.bounds(*args, fw, bw)
    worst = {}
    for k in ("ddsc0", "ddsc1", "dscr0", "dscr1", "ddustbin"):
        if bw.get(k) is None or grads.get(k) is None:
            continue
        got = grads[k] if grads[k] is not None else torch.zeros_like(bw[k])
        worst[k] = mgc.check(f"{label}/{k}", got, bw[k], bnd[k])
        RATIOS[k] = max(RATIOS.get(k, 0.0), worst[k])
    print(label, {k: f"{v:.3f}" for k, v in worst.items()})
    return fw, bw, bnd


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_backward_against_fp64(case):
    B, N, T, dust, g, scale, pitch = case
    args = mgc.case_inputs(B, N, T, dust, g, scale=scale, pitch=pitch, seed=N + B, device=DEV)
    _, grads = run(args)
    compare(_ids(case), args, grads)


def test_backward_without_kp_scores():
    """scr omitted: scores alone, kp = 1, no dscr."""
    args = list(mgc.case_inputs(3, 257, 0.1, True, "s", scr=False, seed=5, device=DEV))
    out, grads = run(args, scr=False)
    assert grads["dscr0"] is None
    compare("noscr", args, grads)


def test_planted_mutations_are_rejected():
    args = mgc.case_inputs(3, 129, 1.0, True, "skf", pitch=160, seed=9, device=DEV)
    _, grads = run(args)
    fw, bw, bnd = compare("mutations", args, grads)
    muts = mgc.mutations(*args, fw)
    assert len(muts) == 5
    for name, out, mutated in muts:
        assert mgc.rejected(bw[out], mutated, bnd[out]), name


def test_deterministic_and_batch_invariant():
    args = mgc.case_inputs(3, 257, 0.1, True, "skf", pitch=288, seed=3, device=DEV)
    _, g1 = run(args)
    _, g2 = run(args)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k
    d0, d1, T, dust, s0, s1, gs, gk, gf = args
    one = [d0[1:2], d1[1:2], T, dust, s0[1:2], s1[1:2], gs[1:2], gk[1:2], gf[1:2]]
    _, ga = run(one)
    for k in ("ddsc0", "ddsc1", "dscr0", "dscr1"):
        assert torch.equal(ga[k][0], g1[k][1]), k


@pytest.fixture(scope="module")
def model_720():
    from mickey_b200.config import mickey_cfg
    from mickey_b200.model import MickeyRelativePose
    from mickey_b200.weights import synthetic_state_dict
    from tests.common import synthetic_pair
    cfg = mickey_cfg("vits", 20, 20)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
    model = model.cuda().eval()
    data = {k: v.to(DEV) for k, v in synthetic_pair(2, 720, 540, seed=17).items()}
    with torch.no_grad():
        model(data)
    return cfg, model, data


def test_forward_equals_the_engine(model_720):
    """On the engine's own descriptors the outputs are bit-identical to model(data)'s (mk_match)."""
    cfg, model, data = model_720
    dust = model.state_dict()[mo.DUSTBIN].to(DEV)
    T = cfg.FEATURE_MATCHER.DUAL_SOFTMAX.TEMPERATURE
    with torch.no_grad():
        sc, kp, fin = dual_softmax(data["dsc0"], data["dsc1"], dust, T, data["scr0"], data["scr1"])
        alone = dual_softmax(data["dsc0"], data["dsc1"], dust, T)
    assert torch.equal(sc, data["scores"]) and torch.equal(kp, data["kp_scores"]) and torch.equal(fin, data["final_scores"])
    assert torch.equal(alone, data["scores"])


def test_training_chain_at_720x540(model_720):
    """Engine features -> dual_softmax with scr -> MetricPoseLoss -> backward(log(final + 1e-16), probs_grad): every
    input gradient within the bounds of the fp64 chain given the same probs_grad; the module drop-in path (torch's kp and
    product) agrees with the fused path."""
    from mickey_b200.loss import MetricPoseLoss
    cfg, model, data = model_720
    t0 = time.time()
    feats = model.extract_features(torch.cat([data["image0"], data["image1"]]))
    B = data["image0"].shape[0]
    dsc, scr = feats.dsc.float(), feats.scr.float()
    N = dsc.shape[-1]
    dsc0, dsc1 = dsc[:B].clone().requires_grad_(), dsc[B:].clone().requires_grad_()
    scr0, scr1 = scr[:B].reshape(B, 1, N).clone().requires_grad_(), scr[B:].reshape(B, 1, N).clone().requires_grad_()
    mm = dualSoftmax(cfg.FEATURE_MATCHER.DUAL_SOFTMAX).to(DEV)
    T = mm.temperature
    sc, kp, fin = dual_softmax(dsc0, dsc1, mm.dustbin_score, T, scr0, scr1)
    batch = {"final_scores": fin.detach(), "kps0": data["kps0"], "kps1": data["kps1"], "depth_kp0": data["depth_kp0"],
             "depth_kp1": data["depth_kp1"], "K_color0": data["K_color0"], "K_color1": data["K_color1"],
             "Kori_color0": data["K_color0"], "Kori_color1": data["K_color1"],
             "T_0to1": loss_cases.planted_pose().float().to(DEV).unsqueeze(0).repeat(B, 1, 1)}
    _, _, (pg,), nv = MetricPoseLoss(loss_cases.loss_cfg(it_matches=20, it_ransac=20))(batch, seed=7)
    assert nv == 1 and bool((pg != 0).any())
    torch.autograd.backward(torch.log(fin + 1e-16), pg)
    fused = {"ddsc0": dsc0.grad, "ddsc1": dsc1.grad, "dscr0": scr0.grad.reshape(B, N), "dscr1": scr1.grad.reshape(B, N),
             "ddustbin": mm.dustbin_score.grad.reshape(())}
    gf = pg / (fin.detach() + 1e-16)
    args = (dsc0.detach(), dsc1.detach(), T, mm.dustbin_score.detach().reshape(1), scr0.detach().reshape(B, N),
            scr1.detach().reshape(B, N), None, None, gf)
    fw, bw, bnd = compare("chain720", args, fused)
    # the module drop-in: the reference's own kp_matrix_scores and product around dualSoftmax
    e0, e1 = dsc0.detach().clone().requires_grad_(), dsc1.detach().clone().requires_grad_()
    r0, r1 = scr0.detach().clone().requires_grad_(), scr1.detach().clone().requires_grad_()
    mm.dustbin_score.grad = None
    scores = mm(e0, e1)
    fin2 = scores * torch.matmul(r0.transpose(2, 1), r1)
    torch.autograd.backward(torch.log(fin2 + 1e-16), pg)
    drop = {"ddsc0": e0.grad, "ddsc1": e1.grad, "dscr0": r0.grad.reshape(B, N), "dscr1": r1.grad.reshape(B, N),
            "ddustbin": mm.dustbin_score.grad.reshape(())}
    for k, v in drop.items():
        assert bool(((v.double() - fused[k].double()).abs() <= 2 * bnd[k] + 1e-30).all()), k
    print(f"training chain B={B} N={N}: {time.time() - t0:.2f} s")


def test_no_grad_and_argument_errors():
    d = torch.nn.functional.normalize(torch.randn(2, 128, 50, device=DEV), dim=1)
    with torch.no_grad():
        s = dual_softmax(d, d, None, 0.1)
    assert s.shape == (2, 50, 50) and not s.requires_grad
    with pytest.raises(ValueError):
        dual_softmax(d, d[:, :, :40], None, 0.1)
    with pytest.raises(ValueError):
        dual_softmax(d, d, torch.tensor([1.0]), 0.1)                        # dustbin on the CPU
    with pytest.raises(ValueError):
        dual_softmax(d, d, None, 0.1, torch.rand(2, 50, device=DEV), None)
    with pytest.raises(ValueError):
        dual_softmax(d, d, None, 0.0)


def test_zz_report_ratios():
    print("max(err / bound):", {k: f"{v:.3f}" for k, v in sorted(RATIOS.items())})
