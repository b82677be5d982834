"""CPU oracle: a plain-PyTorch (CPU, fp32 or fp64) restatement of the reference's inference hot path.

THIS IS TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
`--impl reference` legs may import it; mickey_b200 (the product) never does.

Parity status: the reference's own tests hold no golden vectors for this path (SURVEY.md §4), so the
oracle is pinned against outputs of the reference itself: tests/golden/make_golden.py imports the
unmodified reference from /root/reference (build container only), runs it on seeded inputs with the
seeded synthetic state dict of mickey_b200.weights, and commits the outputs under tests/golden/;
tests/test_oracle_golden.py checks this file against them (and, when /root/reference is present,
against the live reference, stage by stage).

Every function cites the reference lines (relative to /root/reference/lib/models/MicKey/) it
restates.  The restatement is functional: weights come from a flat state dict with the reference's
tensor names (prefix 'compute_matches.extractor.' etc.), nothing here subclasses nn.Module.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
EXTRACTOR = "compute_matches.extractor."
BACKBONE = EXTRACTOR + "dinov2_vitl14."       # name kept by the reference for every variant
DUSTBIN = "compute_matches.matcher.matching_mat.dustbin_score"
VARIANT_HEADS = {384: 6, 768: 12, 1024: 16}    # dinov2.py:306-342 (head_dim is 64 for all)


# ------------------------------------------------------------------------------------------------
# a4 / a8: tokens = patch-embed + cls + interpolated pos-embed
# ------------------------------------------------------------------------------------------------
def interpolate_pos_embed(pos_embed: Tensor, tok_h: int, tok_w: int) -> Tensor:
    """modules/DINO_modules/dinov2.py:165-189.  pos_embed [1, 1+G*G, D] -> [1, 1+tok_h*tok_w, D].

    The reference calls this with (w, h) = (image rows, image cols) (dinov2.py:192 swaps the names),
    adds 0.1 to each token count and resizes the G×G grid bicubically with `scale_factor`."""
    n_grid = pos_embed.shape[1] - 1
    g = int(math.sqrt(n_grid))
    dim = pos_embed.shape[-1]
    if tok_h * tok_w == n_grid and tok_h == tok_w:
        return pos_embed
    pe = pos_embed.float()
    grid = pe[:, 1:].reshape(1, g, g, dim).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, scale_factor=((tok_h + 0.1) / g, (tok_w + 0.1) / g), mode="bicubic")
    assert grid.shape[-2] == tok_h and grid.shape[-1] == tok_w
    grid = grid.permute(0, 2, 3, 1).reshape(1, tok_h * tok_w, dim)
    return torch.cat([pe[:, :1], grid], dim=1).to(pos_embed.dtype)


def vit_tokens(sd: Dict[str, Tensor], img: Tensor) -> Tensor:
    """dinov2.py:191-200 + layers/patch_embed.py:69-82.  img [B,3,H,W] (H,W multiples of 14)."""
    w = sd[BACKBONE + "patch_embed.proj.weight"]
    b = sd[BACKBONE + "patch_embed.proj.bias"]
    p = w.shape[-1]
    B, _, H, W = img.shape
    x = F.conv2d(img, w, b, stride=p)                       # [B, D, H/p, W/p]
    x = x.flatten(2).transpose(1, 2)                        # [B, N, D]
    cls = sd[BACKBONE + "cls_token"].expand(B, -1, -1)
    x = torch.cat([cls, x], dim=1)
    return x + interpolate_pos_embed(sd[BACKBONE + "pos_embed"], H // p, W // p)


# ------------------------------------------------------------------------------------------------
# a5 / a6 / a7: one ViT block
# ------------------------------------------------------------------------------------------------
def vit_attention(sd, pre: str, x: Tensor, heads: int) -> Tensor:
    """layers/attention.py:49-62 (the eager path; MemEffAttention :65-69 falls back to it)."""
    B, T, D = x.shape
    hd = D // heads
    qkv = F.linear(x, sd[pre + "qkv.weight"], sd[pre + "qkv.bias"])
    qkv = qkv.reshape(B, T, 3, heads, hd).permute(2, 0, 3, 1, 4)        # [3,B,h,T,hd]
    q, k, v = qkv[0] * hd ** -0.5, qkv[1], qkv[2]
    att = (q @ k.transpose(-2, -1)).softmax(dim=-1)
    out = (att @ v).transpose(1, 2).reshape(B, T, D)
    return F.linear(out, sd[pre + "proj.weight"], sd[pre + "proj.bias"])


def vit_mlp(sd, pre: str, x: Tensor) -> Tensor:
    """layers/mlp.py:35-41 (exact-erf GELU)."""
    h = F.gelu(F.linear(x, sd[pre + "fc1.weight"], sd[pre + "fc1.bias"]))
    return F.linear(h, sd[pre + "fc2.weight"], sd[pre + "fc2.bias"])


def vit_block(sd, pre: str, x: Tensor, heads: int) -> Tensor:
    """layers/block.py:105-106 (eval branch) with LayerScale (layers/layer_scale.py:27-28)."""
    D = x.shape[-1]
    h = F.layer_norm(x, (D,), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"], eps=1e-6)
    x = x + sd[pre + "ls1.gamma"] * vit_attention(sd, pre + "attn.", h, heads)
    h = F.layer_norm(x, (D,), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"], eps=1e-6)
    x = x + sd[pre + "ls2.gamma"] * vit_mlp(sd, pre + "mlp.", h)
    return x


def vit_forward_features(sd, img: Tensor) -> Tensor:
    """dinov2.py:221-236 -> 'x_norm_patchtokens' [B, N, D]."""
    x = vit_tokens(sd, img)
    D = x.shape[-1]
    heads = VARIANT_HEADS[D]
    depth = 1 + max(int(k.split(".")[4]) for k in sd if k.startswith(BACKBONE + "blocks."))
    for i in range(depth):
        x = vit_block(sd, f"{BACKBONE}blocks.{i}.", x, heads)
    x = F.layer_norm(x, (D,), sd[BACKBONE + "norm.weight"], sd[BACKBONE + "norm.bias"], eps=1e-6)
    return x[:, 1:]


# ------------------------------------------------------------------------------------------------
# a9: residual conv blocks of the heads
# ------------------------------------------------------------------------------------------------
def _bn_eval(sd, pre: str, x: Tensor) -> Tensor:
    return F.batch_norm(x, sd[pre + "running_mean"], sd[pre + "running_var"],
                        sd[pre + "weight"], sd[pre + "bias"], training=False, eps=1e-5)


def basic_block(sd, pre: str, x: Tensor, relu: bool = True, bn: bool = True) -> Tensor:
    """modules/utils/extractor_utils.py:28-35."""
    sc_key = pre + "shortcut.0.weight"
    shortcut = F.conv2d(x, sd[sc_key]) if sc_key in sd else x
    out = F.conv2d(x, sd[pre + "conv1.weight"], padding=1)
    out = F.relu(_bn_eval(sd, pre + "bn1.", out) if bn else out)
    out = F.conv2d(out, sd[pre + "conv2.weight"], padding=1)
    out = (_bn_eval(sd, pre + "bn2.", out) if bn else out) + shortcut
    return F.relu(out) if relu else out


# ------------------------------------------------------------------------------------------------
# a10: linear-attention transformer inside each head
# ------------------------------------------------------------------------------------------------
def sine_position_encoding(d_model: int, h: int, w: int, dtype=torch.float32, device=None) -> Tensor:
    """modules/att_layers/transformer.py:25-36: [d_model, h, w]; positions start at 1."""
    y = torch.arange(1, h + 1, dtype=torch.float32).view(1, h, 1).expand(1, h, w)
    x = torch.arange(1, w + 1, dtype=torch.float32).view(1, 1, w).expand(1, h, w)
    div = torch.exp(torch.arange(0, d_model // 2, 2).float() * (-math.log(10000.0) / (d_model // 2)))
    div = div[:, None, None]
    pe = torch.zeros(d_model, h, w)
    pe[0::4] = torch.sin(x * div)
    pe[1::4] = torch.cos(x * div)
    pe[2::4] = torch.sin(y * div)
    pe[3::4] = torch.cos(y * div)
    return pe.to(dtype).to(device) if device is not None else pe.to(dtype)


def linear_attention(q: Tensor, k: Tensor, v: Tensor, eps: float = 1e-6) -> Tensor:
    """modules/att_layers/attention.py:46-64.  q,k,v [B, L, H, d]."""
    Q = F.elu(q) + 1
    K = F.elu(k) + 1
    n = v.shape[1]
    kv = torch.einsum("bshd,bshv->bhdv", K, v / n)
    z = 1.0 / (torch.einsum("blhd,bhd->blh", Q, K.sum(dim=1)) + eps)
    return torch.einsum("blhd,bhdv,blh->blhv", Q, kv, z) * n


def encoder_layer(sd, pre: str, x: Tensor, nhead: int = 8) -> Tensor:
    """modules/att_layers/transformer_utils.py:40-66 with source == x (self attention)."""
    B, L, C = x.shape
    d = C // nhead
    q = F.linear(x, sd[pre + "q_proj.weight"]).view(B, L, nhead, d)
    k = F.linear(x, sd[pre + "k_proj.weight"]).view(B, L, nhead, d)
    v = F.linear(x, sd[pre + "v_proj.weight"]).view(B, L, nhead, d)
    msg = linear_attention(q, k, v).reshape(B, L, C)
    msg = F.linear(msg, sd[pre + "merge.weight"])
    msg = F.layer_norm(msg, (C,), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"], eps=1e-5)
    msg = F.linear(F.relu(F.linear(torch.cat([x, msg], dim=2), sd[pre + "mlp.0.weight"])),
                   sd[pre + "mlp.2.weight"])
    msg = F.layer_norm(msg, (C,), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"], eps=1e-5)
    return x + msg


def head_transformer(sd, pre: str, x: Tensor, add_pos_enc: bool) -> Tensor:
    """modules/att_layers/transformer.py:75-103 (3 'self' layers, linear attention, 8 heads)."""
    B, C, H, W = x.shape
    if add_pos_enc:
        x = x + sine_position_encoding(C, H, W, x.dtype, x.device)[None]
    t = x.flatten(2).transpose(1, 2)
    n_layers = 1 + max(int(k[len(pre + "layers."):].split(".")[0]) for k in sd if k.startswith(pre + "layers."))
    for i in range(n_layers):
        t = encoder_layer(sd, f"{pre}layers.{i}.", t)
    return t.transpose(1, 2).reshape(B, C, H, W)


def head_trunk(sd, pre: str, feat: Tensor, add_pos_enc: bool, last_relu: bool, bn: bool = True) -> Tensor:
    """Shared body of the four heads: mickey_extractor.py:126-131 / 164-170 / 203-209 / 240-246."""
    x = basic_block(sd, pre + "resblock1.", feat, bn=bn)
    x = basic_block(sd, pre + "resblock2.", x, bn=bn)
    x = basic_block(sd, pre + "resblock3.", x, bn=bn)
    x = head_transformer(sd, pre + "att_layer.", x, add_pos_enc)
    return basic_block(sd, pre + "resblock4.", x, relu=last_relu, bn=bn)


# ------------------------------------------------------------------------------------------------
# a11: output activations
# ------------------------------------------------------------------------------------------------
def score_activation(raw: Tensor, use_softmax: bool, border: int = 3, temp: float = 100.0,
                     eps: float = 1e-16) -> Tensor:
    """mickey_extractor.py:98-124,137-142.  raw [B,1,H,W]."""
    B = raw.shape[0]
    mask = torch.zeros_like(raw)
    mask[:, :, border:raw.shape[2] - border, border:raw.shape[3] - border] = 1
    if not use_softmax:
        return torch.sigmoid(raw) * mask
    s = raw - (raw.reshape(B, -1).mean(-1).view(B, 1, 1, 1) + eps)
    e = torch.exp(s / temp) * mask
    return e / (e.sum(dim=(2, 3), keepdim=True) + eps)


def l2_normalize_channels(d: Tensor, eps: float = 1e-10) -> Tensor:
    """modules/utils/extractor_utils.py:6-10."""
    return d / (d.pow(2).sum(dim=1, keepdim=True) + eps).sqrt()


def extractor(sd, img: Tensor, cfg) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """mickey_extractor.py:43-58 -> (offsets [B,2,h,w], depth [B,1,h,w], score [B,1,h,w], desc [B,128,h,w]).

    The oracle always runs the backbone in the dtype of `img`/`sd` (fp32 by default): it restates the
    reference with FLOAT16: False, the comparator named in DESIGN.md."""
    m = cfg["MICKEY"]
    f = m["DINOV2"]["DOWN_FACTOR"]
    B, _, H, W = img.shape
    img = img[:, :, : f * (H // f), : f * (W // f)]
    # FLOAT16: True (mickey_extractor.py:31-35,49) == backbone weights stored in fp16: the image is cast to the
    # backbone's dtype and the patch tokens come back as fp32 (used by bench.py's eager-CUDA comparator), or as fp64
    # when the heads' weights are fp64
    wdt = sd[BACKBONE + "patch_embed.proj.weight"].dtype
    hdt = torch.float64 if sd[EXTRACTOR + "det_head.resblock1.conv1.weight"].dtype == torch.float64 else torch.float32
    tok = vit_forward_features(sd, img.to(wdt)).to(hdt)
    feat = tok.permute(0, 2, 1).reshape(B, -1, H // f, W // f)
    kp, ds = m["KP_HEADS"], m["DSC_HEAD"]
    bn = kp["BN"]
    score_raw = F.conv2d(head_trunk(sd, EXTRACTOR + "det_head.", feat, kp["POS_ENCODING"], True, bn),
                         sd[EXTRACTOR + "det_head.score.weight"])
    score = score_activation(score_raw, kp["USE_SOFTMAX"])
    offs = torch.sigmoid(F.conv2d(head_trunk(sd, EXTRACTOR + "det_offset.", feat, kp["POS_ENCODING"], True, bn),
                                  sd[EXTRACTOR + "det_offset.xy_offset.weight"]))
    depth = F.conv2d(head_trunk(sd, EXTRACTOR + "depth_head.", feat, kp["POS_ENCODING"], True, bn),
                     sd[EXTRACTOR + "depth_head.depth.weight"])
    if kp["USE_DEPTHSIGMOID"]:
        depth = kp["MAX_DEPTH"] * torch.sigmoid(depth)
    desc = head_trunk(sd, EXTRACTOR + "dsc_head.", feat, ds["POS_ENCODING"], False, bn)
    if ds["NORM_DSC"]:
        desc = l2_normalize_channels(desc)
    return offs, depth, score, desc


# ------------------------------------------------------------------------------------------------
# a12: dual-softmax matcher;  a2: correspondences;  a1: final scores
# ------------------------------------------------------------------------------------------------
def dual_softmax(dsc0: Tensor, dsc1: Tensor, temperature: float, dustbin: Optional[Tensor]) -> Tensor:
    """modules/utils/feature_matcher.py:64-83.  dsc [B,C,N] -> [B,N0,N1]."""
    s = torch.matmul(dsc0.transpose(1, 2), dsc1) / temperature
    if dustbin is None:
        return F.softmax(s, 1) * F.softmax(s, 2)
    b, m, n = s.shape
    full = s.new_empty(b, m + 1, n + 1)
    full[:, :m, :n] = s
    full[:, m, :] = dustbin
    full[:, :, n] = dustbin
    full = F.softmax(full, 1) * F.softmax(full, 2)
    return full[:, :m, :n]


def absolute_keypoints(offsets: Tensor, down_factor: int) -> Tensor:
    """modules/compute_correspondences.py:20-31: (offset + (x, y) cell index) * 14."""
    B, _, H, W = offsets.shape
    xs = torch.arange(W, dtype=offsets.dtype, device=offsets.device).view(1, 1, 1, W).expand(B, 1, H, W)
    ys = torch.arange(H, dtype=offsets.dtype, device=offsets.device).view(1, 1, H, 1).expand(B, 1, H, W)
    return (offsets + torch.cat([xs, ys], dim=1)) * down_factor


def compute_correspondences(sd, data: dict, cfg) -> dict:
    """modules/compute_correspondences.py:52-92 + compute_pose.py:23.  Returns the dict of outputs."""
    f = cfg["MICKEY"]["DINOV2"]["DOWN_FACTOR"]
    out = {}
    per_image = []
    for key in ("image0", "image1"):
        offs, depth, score, desc = extractor(sd, data[key], cfg)
        kps = absolute_keypoints(offs, f)
        B, _, H, W = kps.shape
        per_image.append((kps.reshape(B, 2, H * W), depth.reshape(B, 1, H * W),
                          score.reshape(B, 1, H * W), desc.reshape(B, -1, H * W), depth, [H, W]))
    (k0, d0, s0, c0, dm0, sh0), (k1, d1, s1, c1, dm1, sh1) = per_image
    mcfg = cfg["FEATURE_MATCHER"]["DUAL_SOFTMAX"]
    dustbin = sd[DUSTBIN] if mcfg["USE_DUSTBIN"] else None
    out.update(kps0=k0, kps1=k1, depth_kp0=d0, depth_kp1=d1, scr0=s0, scr1=s1, dsc0=c0, dsc1=c1,
               depth0_map=dm0, depth1_map=dm1, kps0_shape=sh0, kps1_shape=sh1, down_factor=f)
    out["scores"] = dual_softmax(c0, c1, mcfg["TEMPERATURE"], dustbin)
    out["kp_scores"] = torch.matmul(s0.transpose(2, 1), s1)           # compute_correspondences.py:46-50
    out["final_scores"] = out["scores"] * out["kp_scores"]            # compute_pose.py:23
    return out


# ------------------------------------------------------------------------------------------------
# a14 / a15 / a16: geometry
# ------------------------------------------------------------------------------------------------
def backproject(uv: Tensor, depth: Tensor, K: Tensor) -> Tensor:
    """modules/utils/training_utils.py:7-22.  uv [M,n,2], depth [M,n,1], K [M,3,3] -> [M,n,3]."""
    uv1 = torch.cat([uv, torch.ones_like(uv[..., :1])], dim=-1)
    return depth * (torch.linalg.inv(K) @ uv1.transpose(2, 1)).transpose(2, 1)


def kabsch(A: Tensor, Bp: Tensor, w: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """modules/loss/solvers.py:3-54.  w=None: unweighted branch (:32-39); w given: the
    use_weights=True,use_mask=True branch (:13-26) used by the refinement."""
    if w is None:
        a_mean = A.mean(dim=1, keepdim=True)
        b_mean = Bp.mean(dim=1, keepdim=True)
        H = (A - a_mean).transpose(1, 2) @ (Bp - b_mean)
    else:
        wn = (w / (w.abs().sum(1, keepdim=True) + 1e-16)).unsqueeze(-1)
        a_mean = (wn * A).sum(1, keepdim=True)
        b_mean = (wn * Bp).sum(1, keepdim=True)
        H = (A - a_mean).transpose(1, 2) @ (w.unsqueeze(-1) * (Bp - b_mean))
    U, _, V = torch.svd(H)
    Z = torch.eye(3, dtype=A.dtype, device=A.device).repeat(A.shape[0], 1, 1)
    Z[:, 2, 2] = torch.sign(torch.linalg.det(U @ V.transpose(1, 2)))
    R = V @ Z @ U.transpose(1, 2)
    t = b_mean - a_mean @ R.transpose(1, 2)
    return R, t


def residual_norm(X: Tensor, Y: Tensor, R: Tensor, t: Tensor) -> Tensor:
    Xt = (R @ X.transpose(2, 1)).transpose(2, 1) + t
    return (((Xt - Y) ** 2).sum(-1) + 1e-6) ** 0.5


def soft_inliers(X, Y, R, t, th: float) -> Tensor:
    """modules/utils/training_utils.py:55-61 -> [M,1]."""
    return torch.sigmoid((5.0 / th) * (th - residual_norm(X, Y, R, t))).sum(-1, keepdim=True)


def hard_inliers(X, Y, R, t, th: float) -> Tensor:
    """modules/utils/training_utils.py:71-75 -> [M,n] in {0,1}."""
    return ((th - residual_norm(X, Y, R, t)) >= 0).to(X.dtype)


# ------------------------------------------------------------------------------------------------
# a13 / a17 / a18: vectorised probabilistic Procrustes RANSAC
# ------------------------------------------------------------------------------------------------
def solve_pose(final_scores: Tensor, kps0: Tensor, depth0: Tensor, kps1: Tensor, depth1: Tensor,
               K0: Tensor, K1: Tensor, cfg, return_inliers: bool = False,
               outer_idx: Optional[Tensor] = None, inner_idx: Optional[Tensor] = None,
               generator: Optional[torch.Generator] = None, trace: Optional[dict] = None):
    """modules/utils/probabilisticProcrustes.py:183-348 (estimate_pose_vectorized).

    outer_idx [B*IT_MATCHES, n_s] / inner_idx [B*IT_MATCHES*IT_RANSAC, 3]: when given they replace
    the two torch.multinomial draws (:231, :251) so that everything downstream is deterministic
    (this is how the CUDA solver is compared bit-for-bit in structure).  `trace`, when a dict, is
    filled with the intermediate tensors (sampled indices, hypothesis scores, winner ...).

    Where it departs from the reference: NUM_SAMPLED_MATCHES is taken from cfg for every shape.  The
    reference hard-codes 2048 when it reshapes the point tensors (:271-272), so for any other value it
    raises inside its try and returns the zero result; this restatement returns the pose the
    algorithm defines.  It is the fp64 comparator of the CUDA solver's whole range (mk_procrustes_solve:
    any multiple of 256 up to 2048); the drop-in solvers accept 2048 only (mickey_b200.model
    check_sampled_matches)."""
    p = cfg["PROCRUSTES"]
    IM, IR, n_s, n_c = p["IT_MATCHES"], p["IT_RANSAC"], p["NUM_SAMPLED_MATCHES"], p["NUM_CORR_3D_3D"]
    B, N, _ = final_scores.shape
    dev = final_scores.device
    K0, K1 = K0.to(final_scores.dtype), K1.to(final_scores.dtype)
    rows = final_scores.reshape(B, N * N)
    try:
        if outer_idx is None:
            tiled = rows.unsqueeze(1).expand(B, IM, N * N).reshape(B * IM, N * N)
            outer_idx = torch.multinomial(tiled, n_s, generator=generator)              # :231
        b_of = torch.arange(B, device=dev).repeat_interleave(IM)                                     # [B*IM]
        i0 = torch.div(outer_idx, N, rounding_mode="trunc")                              # :233
        i1 = outer_idx % N                                                               # :234
        bb = b_of[:, None].expand(-1, n_s)
        uv0 = kps0[bb, :, i0]                                                            # [B*IM,n_s,2]
        uv1 = kps1[bb, :, i1]
        z0 = depth0[bb, :, i0]                                                           # [B*IM,n_s,1]
        z1 = depth1[bb, :, i1]
        wts = rows[bb, outer_idx]                                                        # :241
        X = backproject(uv0, z0, K0[b_of])                                               # :243
        Y = backproject(uv1, z1, K1[b_of])
        if inner_idx is None:
            wv = wts.unsqueeze(1).expand(B * IM, IR, n_s).reshape(B * IM * IR, n_s)
            inner_idx = torch.multinomial(wv, n_c, generator=generator)                  # :251
        s_of = torch.arange(B * IM, device=dev).repeat_interleave(IR)                                # hypothesis -> set
        Xk = X[s_of[:, None], inner_idx]                                                 # [M,3,3]
        Yk = Y[s_of[:, None], inner_idx]
        R, t = kabsch(Xk, Yk)                                                            # :259
        invalid = bool(torch.isnan(t).any() or torch.isinf(t).any() or
                       torch.isnan(R).any() or torch.isinf(R).any())                     # :261-262
        score = soft_inliers(X[s_of], Y[s_of], R, t, p["TH_SOFT_INLIER"]).reshape(B, IM * IR)   # :265
        best = torch.argmax(score, dim=1)                                                # :275
        bi = torch.arange(B, device=dev)
        R = R.reshape(B, IM * IR, 3, 3)[bi, best]
        t = t.reshape(B, IM * IR, 1, 3)[bi, best]
        best_set = bi * IM + torch.div(best, IR, rounding_mode="trunc")
        Xb, Yb = X[best_set], Y[best_set]
        mask_ref = torch.zeros(B, n_s, dtype=X.dtype, device=dev)
        prev = n_c * torch.ones(B, dtype=X.dtype, device=dev)                                        # :285
        n_ref_done = 0
        for _ in range(p["NUM_REFINEMENTS"]):                                            # :286-300
            inl = hard_inliers(Xb, Yb, R, t, p["TH_INLIER"])
            cnt = inl.sum(-1)
            do = (cnt >= n_c) & (cnt > prev)
            prev = torch.where(do, cnt, prev)
            if not bool(do.any()):
                break
            mask_ref[do] = inl[do]
            R2, t2 = kabsch(Xb[do], Yb[do], mask_ref[do])
            R = R.clone(); t = t.clone()
            R[do], t[do] = R2, t2
            n_ref_done += 1
        inliers = soft_inliers(Xb, Yb, R, t, p["TH_INLIER"])                              # :303
        inl_list = [torch.zeros(0, 5)] * B
        if return_inliers:                                                               # :305-327
            hard = hard_inliers(Xb, Yb, R, t, p["TH_INLIER"])
            inl_list = []
            for b in range(B):
                sel = hard[b] == 1.0
                sset = best_set[b]
                w_b = wts[sset][sel]
                order = torch.argsort(w_b, descending=True)
                inl_list.append(torch.cat([uv0[sset][sel][order], uv1[sset][sel][order],
                                           w_b[order].unsqueeze(-1), z0[sset][sel][order],
                                           z1[sset][sel][order]], dim=1))
        if trace is not None:
            trace.update(outer_idx=outer_idx, inner_idx=inner_idx, X=X, Y=Y, weights=wts,
                         hyp_scores=score, best=best, best_set=best_set, n_refinements=n_ref_done)
        if invalid:
            raise FloatingPointError("invalid hypothesis")
    except Exception:                                                                    # :331-342
        R = torch.zeros(B, 3, 3, device=dev); t = torch.zeros(B, 1, 3, device=dev); inliers = torch.zeros(B, device=dev)
        inl_list = [torch.zeros(0, 5)] * B
    if return_inliers:
        return R, t, inliers, inl_list
    return R, t, inliers


def model_forward(sd, data: dict, cfg, return_inliers: bool = False, **solver_kw):
    """compute_pose.py:20-37.  Fills `data` like the reference does and returns (R, t)."""
    data.update(compute_correspondences(sd, data, cfg))
    res = solve_pose(data["final_scores"], data["kps0"], data["depth_kp0"], data["kps1"],
                     data["depth_kp1"], data["K_color0"].float(), data["K_color1"].float(), cfg,
                     return_inliers=return_inliers, **solver_kw)
    data["R"], data["t"], data["inliers"] = res[0], res[1], res[2]
    if return_inliers:
        data["inliers_list"] = res[3]
    return res[0], res[1]
