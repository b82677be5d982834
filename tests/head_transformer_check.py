"""Element-wise bounds for the heads' transformer (csrc/head_transformer.cu) against fp64, and the planted mutations the
bounds must reject.

`restate` is the forward and the closed-form backward of Transformer_self_att (DESIGN.md §6g) written out stage by stage.
Run in fp64 it is the reference (it equals fp64 autograd of oracle.mickey_oracle.head_transformer, which
tests/test_head_transformer_host.py checks); run in fp32 on the CPU it is a second fp32 implementation the bounds must
accept.  Alongside every fp64 value it carries a first-order running-error estimate e (elementwise, >= 0), built from the
operations the kernels perform, with u = 2^-24:

* a contraction of K products in any order, operands carrying errors ea, eb:
      e = sqrt(sum ea^2 b^2) + sqrt(sum a^2 eb^2) + (K + 2) u sum |a b|
  The last term, the contraction's own rounding (K roundings of the sum, the product, the store), is a worst-case bound.
  The errors its operands carry are combined root-sum-square: they come from independent roundings of earlier stages,
  and the worst case sum |ea| |b| multiplies them by sum_k |W_jk| (about 10 for these weights) at every one of the 15
  contractions of a 3-layer forward and backward, which gives no usable bound.  So the whole is an error model, exact in
  its per-stage rounding terms and statistical in how earlier errors combine; it is not a proof.
* phi(t) = t + 1 (t > 0) or e^t (expf: 2 ulp):  e = min(phi, 1) e_t + 2 u |phi|;  elu'(t) = min(phi(t), 1)
* Z = 1 / den:  e_Z = Z (e_den / den + u)
* LayerNorm of a row a with errors e_a (mu, d = a - mu, sigma^2 = mean d^2, r = (sigma^2 + eps)^-1/2, xhat = d r):
      e_mu = mean e_a + D u mean |a|,  e_d = e_a + e_mu + u |d|,  e_s2 = 2 mean(|d| e_d) + (D + 2) u sigma^2
      e_r = r (e_s2 / (2 (sigma^2 + eps)) + 2 u),  e_xhat = r e_d + |d| e_r + u |xhat|,
      y = gamma xhat + beta:  e_y = |gamma| e_xhat + 2 u (|gamma xhat| + |beta|)
* LayerNorm backward, dz = r (gg - mean gg - xhat mean(gg xhat)), gg = gamma g: the same rules term by term
* ReLU: 1-Lipschitz forward; in the backward an element whose pre-activation lies within its own error of 0 may take
  either side of the mask, so its bound there is |dh| + e
* sums over tokens (S, Ksum, dS, dKsum, dW, dgamma, dbeta): the contraction rule with K = the additions on the longest
  path of the kernels' two-level order, tile + number of tiles (32-token slots per image for the attention sums, 512-token
  slots for dW, 64-token blocks for dgamma and dbeta), folded slot by slot.

The bounds are first order in u.  `SLACK` = 2 covers the second-order terms and the products of two carried errors the
first-order rule drops; it is a fixed allowance, not fitted to observed errors.
"""
from __future__ import annotations

import torch

U = 2.0 ** -24
SLACK = 2.0
LN_EPS = 1e-5
ATT_EPS = 1e-6
D = 128
NH, DH = 8, 16
NAMES = ("q_proj", "k_proj", "v_proj", "merge", "mlp0", "mlp2", "norm1_w", "norm1_b", "norm2_w", "norm2_b")
MUTATIONS = ("kv_drop_tile", "kv_neighbour", "pe_next", "ln_mean_drop", "relu_shift", "elu_one", "dw_drop_tile",
             "out_chunk")
ATT_TILE = 32       # tokens per attention slot of the kernels
W_TILE = 512        # tokens per weight-gradient slot
LN_TILE = 64        # tokens per LayerNorm-gradient slot (8 warps of 8 tokens)


def _two_level(n, tile):
    """Additions on the longest path of a sum of n terms taken in slots of `tile`, then folded slot by slot."""
    return min(n, tile) + -(-n // tile)


def _rss(spec, e, v, swap=False):
    """A carried error through a contraction: root-sum-square over the contracted index (see the module docstring)."""
    return (torch.einsum(spec, v * v, e * e) if swap else torch.einsum(spec, e * e, v * v)).sqrt()


def _mm(a, ea, b, eb, K):
    """a [.., K] @ b [K, n] with carried errors (b exact or carrying eb)."""
    v = a @ b
    e = ((ea * ea) @ (b * b)).sqrt() + ((a * a) @ (eb * eb)).sqrt() + (K + 2) * U * (a.abs() @ b.abs())
    return v, e


def _phi(t, et):
    p = torch.where(t > 0, t + 1, torch.exp(t))
    return p, torch.clamp(p, max=1) * et + 2 * U * p.abs()


def _ln(a, ea, gamma, beta):
    mu = a.mean(-1, keepdim=True)
    e_mu = ea.mean(-1, keepdim=True) + D * U * a.abs().mean(-1, keepdim=True)
    d = a - mu
    e_d = ea + e_mu + U * d.abs()
    s2 = (d * d).mean(-1, keepdim=True)
    e_s2 = 2 * (d.abs() * e_d).mean(-1, keepdim=True) + (D + 2) * U * s2
    r = (s2 + LN_EPS).rsqrt()
    e_r = r * (e_s2 / (2 * (s2 + LN_EPS)) + 2 * U)
    xh = d * r
    e_xh = r * e_d + d.abs() * e_r + U * xh.abs()
    y = gamma * xh + beta
    e_y = gamma.abs() * e_xh + 2 * U * ((gamma * xh).abs() + beta.abs())
    return y, e_y, xh, e_xh, r, e_r


def _ln_bwd(g, eg, xh, e_xh, r, e_r, gamma, mutate_mean=False):
    gg = gamma * g
    e_gg = gamma.abs() * eg + U * gg.abs()
    m1 = gg.mean(-1, keepdim=True)
    e_m1 = e_gg.mean(-1, keepdim=True) + D * U * gg.abs().mean(-1, keepdim=True)
    m2 = (gg * xh).mean(-1, keepdim=True)
    e_m2 = (e_gg * xh.abs() + gg.abs() * e_xh).mean(-1, keepdim=True) + (D + 1) * U * (gg * xh).abs().mean(-1, keepdim=True)
    inner = gg - (0 if mutate_mean else m1) - xh * m2
    e_in = e_gg + e_m1 + e_xh * m2.abs() + xh.abs() * e_m2 + 3 * U * (gg.abs() + m1.abs() + (xh * m2).abs())
    dz = r * inner
    e_dz = e_r * inner.abs() + r * e_in + U * dz.abs()
    T = g.shape[0]
    dgam = (g * xh).sum(0)
    e_dgam = (eg * xh.abs() + g.abs() * e_xh).sum(0) + (_two_level(T, LN_TILE) + 2) * U * (g * xh).abs().sum(0)
    dbet = g.sum(0)
    e_dbet = eg.sum(0) + (_two_level(T, LN_TILE) + 1) * U * g.abs().sum(0)
    return dz, e_dz, dgam, e_dgam, dbet, e_dbet


def _dw(dy, edy, x, ex, drop_last=False):
    """dW = dy^T x over tokens; drop_last drops the last weight-gradient slot."""
    if drop_last:
        keep = ((dy.shape[0] - 1) // W_TILE) * W_TILE
        dy, x = dy[:keep], x[:keep]
        edy, ex = edy[:keep], ex[:keep]
    T = dy.shape[0]
    v = dy.t() @ x
    e = ((edy * edy).t() @ (x * x)).sqrt() + ((dy * dy).t() @ (ex * ex)).sqrt() + (_two_level(T, W_TILE) + 2) * U * (dy.abs().t() @ x.abs())
    return v, e


def restate(x, params, pe, grad_out, mutation=None, dtype=torch.float64, x_err=None, grad_err=None):
    """Forward and backward of the transformer.  x, grad_out [B, 128, h, w]; params: 10 per layer (NAMES order); pe:
    the positional encoding [1, 128, 256, 256] or None.  Returns {name: (value, bound)} for 'out', 'dx' and
    'L{i}.{name}' (the parameters' gradients); the bounds are those of an fp32 implementation against the fp64 values
    (meaningful with dtype = float64).  x_err / grad_err [B, 128, h, w]: errors the fp32 implementation's x and grad_out
    already carry (an fp32 layer in front of it or behind it), None = exact.  `mutation` plants one of MUTATIONS in the
    values (not the bounds)."""
    B, C, h, w = x.shape
    N = h * w
    T = B * N
    L = len(params) // 10
    cv = lambda t: t.detach().to(dtype).cpu()
    P = [cv(p) for p in params]
    xin = cv(x)
    if pe is not None:
        shift = 1 if mutation == "pe_next" else 0
        pes = cv(pe)[0][:, :h, shift:w + shift]
        xin = xin + pes
    t = xin.reshape(B, C, N).transpose(1, 2).reshape(T, C)
    et = (U * t.abs()) if pe is not None else torch.zeros_like(t)
    if x_err is not None:
        et = et + cv(x_err).reshape(B, C, N).transpose(1, 2).reshape(T, C)
    zero = lambda a: torch.zeros_like(a)
    saved = []
    for l in range(L):
        Wq, Wk, Wv, Wm, W0, W2, g1, b1, g2, b2 = P[10 * l:10 * l + 10]
        Wqkv = torch.cat([Wq, Wk, Wv], 0)
        qkv, e_qkv = _mm(t, et, Wqkv.t(), zero(Wqkv.t()), D)
        pq, e_pq = _phi(qkv[:, :D], e_qkv[:, :D])
        pk, e_pk = _phi(qkv[:, D:2 * D], e_qkv[:, D:2 * D])
        v, e_v = qkv[:, 2 * D:], e_qkv[:, 2 * D:]
        hq = lambda a: a.reshape(B, N, NH, DH)
        Q, K, V = hq(pq), hq(pk), hq(v)
        eQ, eK, eV = hq(e_pq), hq(e_pk), hq(e_v)
        Kk, Vk, eKk, eVk = K, V, eK, eV
        if mutation == "kv_drop_tile" and l == 0:
            keep = torch.ones(B, N, 1, 1, dtype=dtype)
            keep[-1, ((N - 1) // ATT_TILE) * ATT_TILE:] = 0
            Kk, Vk = K * keep, V * keep
        S = torch.einsum("bshd,bshv->bhdv", Kk, Vk)
        e_S = _rss("bshd,bshv->bhdv", eKk, Vk) + _rss("bshd,bshv->bhdv", eVk, Kk, swap=True) + \
            (_two_level(N, ATT_TILE) + 2) * U * torch.einsum("bshd,bshv->bhdv", Kk.abs(), Vk.abs())
        Ks = Kk.sum(1)
        e_Ks = eKk.sum(1) + (_two_level(N, ATT_TILE) + 1) * U * Kk.abs().sum(1)
        if mutation == "kv_neighbour" and l == 0 and B >= 2:
            S, Ks = S.clone(), Ks.clone()
            S[-1], Ks[-1] = S[-2], Ks[-2]
        den = torch.einsum("blhd,bhd->blh", Q, Ks) + ATT_EPS
        e_den = _rss("blhd,bhd->blh", eQ, Ks) + _rss("blhd,bhd->blh", e_Ks, Q, swap=True) + \
            (DH + 2) * U * torch.einsum("blhd,bhd->blh", Q.abs(), Ks.abs())
        Z = 1 / den
        e_Z = Z * (e_den / den + U)
        wv = torch.einsum("blhd,bhdv->blhv", Q, S)
        e_w = _rss("blhd,bhdv->blhv", eQ, S) + _rss("blhd,bhdv->blhv", e_S, Q, swap=True) + \
            (DH + 2) * U * torch.einsum("blhd,bhdv->blhv", Q.abs(), S.abs())
        msg = (Z[..., None] * wv)
        e_msg = e_Z[..., None] * wv.abs() + Z[..., None] * e_w + U * msg.abs()
        msg2, e_msg2 = msg.reshape(T, D), e_msg.reshape(T, D)
        a, e_a = _mm(msg2, e_msg2, Wm.t(), zero(Wm.t()), D)
        m1, e_m1, xh1, e_xh1, r1, e_r1 = _ln(a, e_a, g1, b1)
        cat, e_cat = torch.cat([t, m1], 1), torch.cat([et, e_m1], 1)
        hp, e_hp = _mm(cat, e_cat, W0.t(), zero(W0.t()), 2 * D)
        hr = hp.clamp(min=0)
        y, e_y = _mm(hr, e_hp, W2.t(), zero(W2.t()), 2 * D)
        m2, e_m2, xh2, e_xh2, r2, e_r2 = _ln(y, e_y, g2, b2)
        out = t + m2
        e_out = et + e_m2 + U * out.abs()
        saved.append(dict(t=t, et=et, pq=pq, e_pq=e_pq, pk=pk, e_pk=e_pk, v=v, e_v=e_v, qpre=qkv, S=S, e_S=e_S, Ks=Ks,
                          e_Ks=e_Ks, Z=Z, e_Z=e_Z, wv=wv, e_w=e_w, msg=msg2, e_msg=e_msg2, xh1=xh1, e_xh1=e_xh1, r1=r1,
                          e_r1=e_r1, cat=cat, e_cat=e_cat, hp=hp, e_hp=e_hp, hr=hr, xh2=xh2, e_xh2=e_xh2, r2=r2, e_r2=e_r2))
        t, et = out, e_out
    res = {}
    o = t.reshape(B, N, C).transpose(1, 2).reshape(B, C, h, w)
    eo = et.reshape(B, N, C).transpose(1, 2).reshape(B, C, h, w)
    if mutation == "out_chunk" and N >= 2:
        o = o.clone()
        o[-1, 32:64, 0, 0] = o.reshape(B, C, N)[-1, 32:64, 1]
    res["out"] = (o, eo)
    if grad_out is None:
        return res
    g = cv(grad_out).reshape(B, C, N).transpose(1, 2).reshape(T, C)
    eg = torch.zeros_like(g) if grad_err is None else cv(grad_err).reshape(B, C, N).transpose(1, 2).reshape(T, C)
    for l in range(L - 1, -1, -1):
        s = saved[l]
        Wq, Wk, Wv, Wm, W0, W2, g1, b1, g2, b2 = P[10 * l:10 * l + 10]
        dy, e_dy, dg2, e_dg2, db2, e_db2 = _ln_bwd(g, eg, s["xh2"], s["e_xh2"], s["r2"], s["e_r2"], g2,
                                                   mutate_mean=(mutation == "ln_mean_drop" and l == L - 1))
        res[f"L{l}.norm2_w"], res[f"L{l}.norm2_b"] = (dg2, e_dg2), (db2, e_db2)
        res[f"L{l}.mlp2"] = _dw(dy, e_dy, s["hr"], s["e_hp"])
        dhf, e_dhf = _mm(dy, e_dy, W2, zero(W2), D)
        mask = s["hp"] > 0
        if mutation == "relu_shift" and l == L - 1:
            mask = torch.roll(mask, 1, dims=1)
        dh = torch.where(mask, dhf, torch.zeros_like(dhf))
        e_dh = torch.where(s["hp"].abs() <= s["e_hp"], dhf.abs() + e_dhf, torch.where(mask, e_dhf, torch.zeros_like(e_dhf)))
        res[f"L{l}.mlp0"] = _dw(dh, e_dh, s["cat"], s["e_cat"], drop_last=(mutation == "dw_drop_tile" and l == L - 1))
        dcat, e_dcat = _mm(dh, e_dh, W0, zero(W0), 2 * D)
        dz, e_dz, dg1, e_dg1, db1, e_db1 = _ln_bwd(dcat[:, D:], e_dcat[:, D:], s["xh1"], s["e_xh1"], s["r1"], s["e_r1"], g1)
        res[f"L{l}.norm1_w"], res[f"L{l}.norm1_b"] = (dg1, e_dg1), (db1, e_db1)
        res[f"L{l}.merge"] = _dw(dz, e_dz, s["msg"], s["e_msg"])
        dmsg, e_dmsg = _mm(dz, e_dz, Wm, zero(Wm), D)
        # linear attention
        hq = lambda a: a.reshape(B, N, NH, DH)
        G, eG = hq(dmsg), hq(e_dmsg)
        Q, eQ, K, eK, V, eV = hq(s["pq"]), hq(s["e_pq"]), hq(s["pk"]), hq(s["e_pk"]), hq(s["v"]), hq(s["e_v"])
        S, e_S, Ks, e_Ks, Z, e_Z, wv, e_w = s["S"], s["e_S"], s["Ks"], s["e_Ks"], s["Z"], s["e_Z"], s["wv"], s["e_w"]
        gw = (G * wv).sum(-1)
        e_gw = (eG * wv.abs() + G.abs() * e_w).sum(-1) + (DH + 2) * U * (G * wv).abs().sum(-1)
        c = -Z * Z * gw
        e_c = 2 * Z * e_Z * gw.abs() + Z * Z * e_gw + 3 * U * c.abs()
        sg = torch.einsum("blhv,bhdv->blhd", G, S)
        e_sg = _rss("blhv,bhdv->blhd", eG, S) + _rss("blhv,bhdv->blhd", e_S, G, swap=True) + \
            (DH + 2) * U * torch.einsum("blhv,bhdv->blhd", G.abs(), S.abs())
        dpq = Z[..., None] * sg + c[..., None] * Ks[:, None]
        e_dpq = e_Z[..., None] * sg.abs() + Z[..., None] * e_sg + e_c[..., None] * Ks[:, None].abs() + \
            c[..., None].abs() * e_Ks[:, None] + 3 * U * ((Z[..., None] * sg).abs() + (c[..., None] * Ks[:, None]).abs())
        elu = lambda p: torch.ones_like(p) if mutation == "elu_one" else p.clamp(max=1)
        delu = lambda p, ep: ep * (p < 1)
        dq = dpq * elu(Q)
        e_dq = e_dpq * Q.clamp(max=1) + dpq.abs() * delu(Q, eQ) + U * dq.abs()
        ZQ = Z[..., None] * Q
        dS = torch.einsum("blhd,blhv->bhdv", ZQ, G)
        e_dS = torch.einsum("blhd,blhv->bhdv", e_Z[..., None] * Q.abs() + Z[..., None] * eQ, G.abs()) + \
            _rss("blhd,blhv->bhdv", eG, ZQ, swap=True) + (_two_level(N, ATT_TILE) + 3) * U * torch.einsum("blhd,blhv->bhdv", ZQ.abs(), G.abs())
        dKs = torch.einsum("blh,blhd->bhd", c, Q)
        e_dKs = _rss("blh,blhd->bhd", e_c, Q) + _rss("blh,blhd->bhd", eQ, c, swap=True) + \
            (_two_level(N, ATT_TILE) + 2) * U * torch.einsum("blh,blhd->bhd", c.abs(), Q.abs())
        dpk = torch.einsum("bhdv,blhv->blhd", dS, V) + dKs[:, None]
        e_dpk = _rss("bhdv,blhv->blhd", e_dS, V) + _rss("bhdv,blhv->blhd", eV, dS, swap=True) + \
            e_dKs[:, None] + (DH + 3) * U * (torch.einsum("bhdv,blhv->blhd", dS.abs(), V.abs()) + dKs[:, None].abs())
        dk = dpk * elu(K)
        e_dk = e_dpk * K.clamp(max=1) + dpk.abs() * delu(K, eK) + U * dk.abs()
        dv = torch.einsum("bhdv,blhd->blhv", dS, K)
        e_dv = _rss("bhdv,blhd->blhv", e_dS, K) + _rss("bhdv,blhd->blhv", eK, dS, swap=True) + \
            (DH + 2) * U * torch.einsum("bhdv,blhd->blhv", dS.abs(), K.abs())
        fl = lambda a: a.reshape(T, D)
        dqkv = torch.cat([fl(dq), fl(dk), fl(dv)], 1)
        e_dqkv = torch.cat([fl(e_dq), fl(e_dk), fl(e_dv)], 1)
        for i, name in enumerate(("q_proj", "k_proj", "v_proj")):
            res[f"L{l}.{name}"] = _dw(dqkv[:, i * D:(i + 1) * D], e_dqkv[:, i * D:(i + 1) * D], s["t"], s["et"])
        Wqkv = torch.cat([Wq, Wk, Wv], 0)
        dx1, e_dx1 = _mm(dqkv, e_dqkv, Wqkv, zero(Wqkv), 3 * D)
        gx = g + dcat[:, :D] + dx1
        egx = eg + e_dcat[:, :D] + e_dx1 + 2 * U * (g.abs() + dcat[:, :D].abs() + dx1.abs())
        g, eg = gx, egx
    res["dx"] = (g.reshape(B, N, C).transpose(1, 2).reshape(B, C, h, w), eg.reshape(B, N, C).transpose(1, 2).reshape(B, C, h, w))
    return {k: (v, SLACK * e) for k, (v, e) in res.items()}


def param_key(i: int) -> str:
    return f"L{i // 10}.{NAMES[i % 10]}"


def where(name: str, idx, shape) -> str:
    """Human-readable position of a flat index of output `name`."""
    coords = list(torch.unravel_index(torch.tensor(idx), shape))
    coords = [int(c) for c in coords]
    if name in ("out", "dx"):
        b, c, y, x = coords
        return f"image {b}, token {y * shape[3] + x} (row {y}, col {x}), channel {c}"
    layer, pname = name.split(".")
    return f"layer {layer[1:]}, {pname}, element {tuple(coords)}"


def check(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """Assert |got - ref| <= bound everywhere; return max(err / bound)."""
    got = got.detach().double().cpu()
    err = (got - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        ratio = torch.where(bad, err / bound.clamp(min=1e-300), torch.zeros_like(err))
        i = int(ratio.reshape(-1).argmax())
        raise AssertionError(f"{name}: {int(bad.sum())} of {err.numel()} elements outside the bound; worst at "
                             f"{where(name, i, err.shape)}: got {got.reshape(-1)[i].item():.9g}, fp64 "
                             f"{ref.reshape(-1)[i].item():.9g}, bound {bound.reshape(-1)[i].item():.3g}")
    return float((err / bound.clamp(min=1e-300)).max())


def rejected(ref: dict, mutated: dict) -> bool:
    """Some output of the mutated reference leaves the bound of the true one."""
    return any(bool(((mutated[k][0] - v).abs() > e).any()) for k, (v, e) in ref.items())


def case_inputs(B, h, w, num_layers, seed=0, device="cpu"):
    """Seeded inputs: a head's feature map scale (unit Gaussian), Xavier-uniform weights as the reference initialises
    them, LayerNorm gamma and beta perturbed away from 1 and 0, and a Gaussian upstream gradient."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, h, w, generator=g)
    params = []
    for _ in range(num_layers):
        for name in NAMES:
            if name in ("mlp0",):
                shape = (2 * D, 2 * D)
            elif name == "mlp2":
                shape = (D, 2 * D)
            elif name.startswith("norm"):
                shape = (D,)
            else:
                shape = (D, D)
            if len(shape) == 2:
                bound = (6.0 / (shape[0] + shape[1])) ** 0.5
                p = (torch.rand(shape, generator=g) * 2 - 1) * bound
            elif name.endswith("_w"):
                p = 1 + 0.2 * torch.randn(shape, generator=g)
            else:
                p = 0.1 * torch.randn(shape, generator=g)
            params.append(p)
    go = torch.randn(B, D, h, w, generator=g)
    return x.to(device), [p.to(device) for p in params], go.to(device)
