"""Plain-torch restatement of MicKey's training loss, MetricPoseLoss.RANSAC_vectorized
(lib/models/MicKey/modules/loss/loss_class.py:79-329), device- and dtype-agnostic, with injectable draws.

It is the reference's algorithm in eager torch: the tests compare mickey_b200/loss.py (CUDA search and gradient,
autograd tail) with it in fp64, tests/golden/make_loss_fixture.py pins it to the live reference, and
tools/loss_bench.py times it as the eager baseline.  The tail's helpers (back-projection, weighted Procrustes, soft
count, VCRE / POSE_ERR) are the torch restatements in mickey_b200/loss.py, which the fixture test pins to the reference
through this module.
"""
import numpy as np
import torch

from mickey_b200.loss import (LossParams, backproject_3d, compute_pose_loss, compute_vcre_loss, soft_inlier_counting_3d,
                              vcre_grid, weighted_procrustes)


def _raise_like_multinomial(rows):
    """torch.multinomial's refusal of a row that sums to zero, decided on the host: on a CUDA device torch reports it
    as a device-side assertion instead of an exception the reference's try/except could catch."""
    if bool((rows.sum(-1) == 0).any()):
        raise RuntimeError("invalid multinomial distribution (sum of probabilities <= 0)")


def _hard_inliers(X, Y, R, t, th):
    """training_utils.py:71-75, plus each entry's margin |th - dist|."""
    d = ((((R @ X.transpose(2, 1)).transpose(2, 1) + t - Y) ** 2.0).sum(-1) + 1e-6) ** 0.5
    return ((th - d) >= 0).to(X.dtype), (th - d).abs()


def refine(X_v, Y_v, inner, p: LossParams):
    """:163-196: the refinement of every hypothesis from its C drawn entries.  Returns (inliers_final [H, S], margin
    [H]: the smallest |INLIER_REF_TH - dist| over the inlier tests that decided the hypothesis's refinement)."""
    H, S = X_v.shape[0], X_v.shape[1]
    dev, dt = X_v.device, X_v.dtype
    rows = torch.arange(H, device=dev).unsqueeze(1).expand_as(inner)
    inliers_pre = p.num_corr * torch.ones(H, dtype=dt, device=dev)
    inliers_ref = torch.zeros(H, S, dtype=dt, device=dev)
    inliers_final = torch.zeros(H, S, dtype=dt, device=dev)
    inliers_final[rows, inner] = 1
    inliers = torch.zeros(H, S, dtype=dt, device=dev)
    inliers[rows, inner] = 1
    do_ref = torch.ones(H, dtype=torch.bool, device=dev)
    margin = torch.full((H,), float("inf"), dtype=dt, device=dev)
    R_d = torch.zeros(H, 3, 3, dtype=dt, device=dev)
    t_d = torch.zeros(H, 1, 3, dtype=dt, device=dev)
    for _ in range(p.num_ref_steps):
        R_d[do_ref], t_d[do_ref] = weighted_procrustes(X_v[do_ref], Y_v[do_ref], inliers[do_ref])
        inl, mg = _hard_inliers(X_v[do_ref], Y_v[do_ref], R_d[do_ref], t_d[do_ref], p.inlier_ref_th)
        inliers_ref[do_ref] = inl
        margin[do_ref] = torch.minimum(margin[do_ref], mg.min(-1).values)
        do_ref = inliers_ref.sum(-1) > inliers_pre
        inliers_pre[do_ref] = inliers_ref.sum(-1)[do_ref]
        inliers_final[do_ref] = inliers[do_ref]
        inliers[do_ref] = inliers_ref[do_ref]
        if int(do_ref.sum()) == 0:
            break
    return inliers_final, margin


def gradients(sampled, loss_value, baseline, mask_topk, B, N, IM):
    """:251-261 and :299-316: the REINFORCE gradient [B, N, N] (sum over iterations in order)."""
    dt, dev = loss_value.dtype, loss_value.device
    g = torch.zeros(B, N * N, dtype=dt, device=dev)
    gb = torch.zeros(B, N * N, dtype=dt, device=dev)
    for s in range(B * IM):
        b = s // IM
        tmp = torch.zeros(N * N, dtype=dt, device=dev)
        tmp[sampled[s]] = 1
        gb[b] += tmp
        g[b] += tmp * loss_value[s]
    g = (g - gb * baseline.view(B, 1)) / IM
    return (g * mask_topk.unsqueeze(-1)).reshape(B, N, N)


def metric_pose_loss(batch, p: LossParams, topK=None, outer_idx=None, inner_idx=None, generator=None, dtype=torch.float64):
    """The whole loss.  Draws: outer_idx [B*IM, S] / inner_idx [B*IM*IR, C] when given, else torch.multinomial (:138,
    :159) with `generator`.  Returns a dict: avg_loss, baseline [B], loss_value [B*IM] (or None), scores [B*IM*IR],
    inliers_final [B*IM*IR, S], margin [B*IM*IR], probs_grad [B, N, N], mask_topk, num_valid_h, sampled, inner, and the
    reference's outputs (kps0 / kps1 / depth0 / depth1 leaves, avg_loss_rot, avg_loss_trans, avg_rot_errs, avg_t_errs)."""
    topK = p.topK if topK is None else topK
    fs = batch["final_scores"].detach().to(dtype)
    B, N = fs.shape[0], fs.shape[1]
    IM, IR, S, Cn = p.it_matches, p.it_ransac, p.n_sample, p.num_corr
    dev = fs.device
    leaf = lambda t: t.detach().to(dtype).requires_grad_()
    kps0, depth0, kps1, depth1 = (leaf(batch[k]) for k in ("kps0", "depth_kp0", "kps1", "depth_kp1"))
    Rgt = batch["T_0to1"][:, :3, :3].to(dtype)
    tgt = batch["T_0to1"][:, :3, 3:].transpose(1, 2).to(dtype)
    K0, K1 = batch["K_color0"].to(dtype), batch["K_color1"].to(dtype)
    Kori0, Kori1 = batch["Kori_color0"].to(dtype), batch["Kori_color1"].to(dtype)
    out = {"kps0": kps0, "kps1": kps1, "depth0": depth0, "depth1": depth1, "loss_value": None, "scores": None,
           "inliers_final": None, "margin": None, "sampled": None, "inner": None}
    rows = fs.reshape(B, N * N)
    baseline = torch.zeros(B, dtype=dtype, device=dev)
    losses_rot = torch.zeros(B, 1, dtype=dtype, device=dev)
    losses_trans = torch.zeros(B, 1, dtype=dtype, device=dev)
    num_valid_h = 0
    invalid = bool(torch.isnan(rows).any() or torch.isinf(rows).any() or (rows < 0).any())       # :126-131
    sampled = None
    if not invalid:
        try:                                                                                      # :134, :269-276
            if outer_idx is None:
                _raise_like_multinomial(rows)
                sampled = torch.multinomial(rows.repeat_interleave(IM, 0).float(), S, generator=generator)
            else:
                sampled = outer_idx.to(dev).long()
            bidx = torch.arange(B, device=dev).repeat_interleave(IM).unsqueeze(1).expand(-1, S)
            i0, i1 = torch.div(sampled, N, rounding_mode="trunc"), sampled % N
            X = backproject_3d(kps0[bidx, :2, i0], depth0[bidx, :2, i0], K0.repeat_interleave(IM, 0))     # :144-152
            Y = backproject_3d(kps1[bidx, :2, i1], depth1[bidx, :2, i1], K1.repeat_interleave(IM, 0))
            w = rows[bidx, sampled]
            X_v = X.unsqueeze(1).expand(-1, IR, -1, -1).reshape(B * IM * IR, S, 3)                          # :155-157
            Y_v = Y.unsqueeze(1).expand(-1, IR, -1, -1).reshape(B * IM * IR, S, 3)
            w_v = w.unsqueeze(1).expand(-1, IR, -1).reshape(B * IM * IR, S)
            _raise_like_multinomial(w_v)
            if inner_idx is None:
                inner = torch.multinomial(w_v.float(), Cn, generator=generator)                            # :159
            else:
                inner = inner_idx.to(dev).long()
            with torch.no_grad():
                inl, margin = refine(X_v.detach(), Y_v.detach(), inner, p)
            out.update(sampled=sampled, inner=inner, inliers_final=inl, margin=margin)
            R, t = weighted_procrustes(X_v, Y_v, inl)                                                       # :199-200
            if bool(torch.isfinite(R).all()) and bool(torch.isfinite(t).all()):                            # :213-223
                score_k = soft_inlier_counting_3d(X_v, Y_v, R, t, p.inlier_3d_th)                           # :226
                rep = IM * IR
                loss_fn = compute_vcre_loss if p.loss_type == "VCRE" else compute_pose_loss
                lv_k, lr_k, lt_k = loss_fn(R, t, Rgt.repeat_interleave(rep, 0), tgt.repeat_interleave(rep, 0),
                                           Kori0.repeat_interleave(rep, 0), Kori1.repeat_interleave(rep, 0),
                                           vcre_grid(dev).to(dtype), p.soft_clipping)                      # :229
                lv_k, lr_k, lt_k, score_k = (x.reshape(B * IM, IR) for x in (lv_k, lr_k, lt_k, score_k))
                out["scores"] = score_k.reshape(-1)
                sm = torch.softmax(score_k / p.score_temperature, -1)                                       # :238-239
                loss_rot, loss_trans = (lr_k * sm).sum(-1), (lt_k * sm).sum(-1)
                if p.add_null_hypothesis:                                                                   # :241-245
                    lv_k = torch.cat([lv_k, torch.full((B * IM, 1), p.max_loss_null, dtype=dtype, device=dev)], -1)
                    score_k = torch.cat([score_k, torch.full((B * IM, 1), p.th_outliers * S, dtype=dtype, device=dev)], -1)
                loss_value = (lv_k * torch.softmax(score_k / p.score_temperature, -1)).sum(-1)             # :248
                out["loss_value"] = loss_value
                losses_rot = loss_rot.reshape(B, IM).sum(-1).unsqueeze(-1)                                  # :263-265
                losses_trans = loss_trans.reshape(B, IM).sum(-1).unsqueeze(-1)
                baseline = loss_value.reshape(B, IM).sum(-1)
                num_valid_h = 1
        except RuntimeError:
            pass
    baseline = baseline / IM                                                                                # :294-296
    losses_trans, losses_rot = losses_trans / IM, losses_rot / IM
    if p.train_w_top and B > 1:                                                                             # :309-319
        select_top_b = np.maximum(int(B * topK / 100), 1)
        topk_loss = baseline[torch.argsort(baseline)[select_top_b]]
        mask_topk = (baseline < topk_loss).to(dtype)
        avg_loss = (mask_topk * baseline).sum() / mask_topk.sum()
    else:
        avg_loss = torch.mean(baseline)
        mask_topk = torch.ones(B, dtype=dtype, device=dev)
    if out["loss_value"] is None:
        probs_grad = torch.zeros(B, N, N, dtype=dtype, device=dev)
    else:
        probs_grad = gradients(sampled, out["loss_value"].detach(), baseline.detach(), mask_topk, B, N, IM)
    out.update(avg_loss=avg_loss, baseline=baseline, probs_grad=probs_grad, mask_topk=mask_topk, num_valid_h=num_valid_h,
               avg_loss_rot=torch.mean(losses_rot), avg_loss_trans=torch.mean(losses_trans),
               avg_rot_errs=torch.mean(torch.rad2deg(losses_rot)), avg_t_errs=torch.mean(losses_trans))
    return out
