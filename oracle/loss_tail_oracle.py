"""The differentiable tail of MicKey's training loss (lib/models/MicKey/modules/loss/loss_class.py:140-152, 199-248) in
closed form, the comparator of csrc/loss_tail.cu (MetricPoseLoss(cfg, cuda_tail=True)).

- tail_autograd: the reference's tail composed from the restated helpers of mickey_b200/loss.py (back-projection,
  weighted Procrustes through torch.svd, soft count, VCRE / POSE_ERR, the softmaxes), differentiable in the four leaves.
- procrustes_backward: dL/dH of the Kabsch rotation without an SVD.
- tail_closed_form: the tail's values and its closed-form backward, the arithmetic the kernels run, with planted
  mutations (TAIL_MUTATIONS) that tests/test_loss_tail_host.py must reject.
"""
import torch

from mickey_b200.loss import (LossParams, backproject_3d, compute_pose_loss, compute_vcre_loss, soft_inlier_counting_3d,
                              vcre_grid, weighted_procrustes)

# planted errors the tests must reject: the first five by tests/test_loss_tail_host.py's 1e-10 comparison with autograd,
# the rest by the element-wise bound of tests/loss_tail_check.py (they are the size of the kernel's own slips):
# ki_fp64 the exact fp64 K^-1 in place of the kernel's fp32 one; vcre_inverse_tgt tgt in place of Rgt Rgt^T tgt;
# vcre_gate_gt the clamp gate on the ground-truth projection; rot_weights_q loss_rot / loss_trans weighted by the
# null-inclusive softmax; scatter_drop_last each keypoint's last contribution in ascending order dropped;
# last_hyp_dropped hypothesis IR - 1 left out of the entry sums; sigmoid_fp32 the soft score's sigmoid in fp32
TAIL_MUTATIONS = ("rt_sign", "z_in_m", "score_direct", "mean_x", "acos_edge", "ki_fp64", "vcre_inverse_tgt",
                  "vcre_gate_gt", "rot_weights_q", "scatter_drop_last", "last_hyp_dropped", "sigmoid_fp32")
ACOS_CLIP = 0.99999


def kernel_kinv(K):
    """K^-1 as csrc/loss_tail.cu back-projects with it: the fp64 inverse of the fp32 K rounded to fp32 (inv3x3), in
    fp64.  [B, 3, 3]."""
    return torch.linalg.inv(K.double()).float().double()


def _set_points(kps0, depth0, kps1, depth1, K0, K1, sampled, IM, Kinv=None):
    """The back-projected X, Y [B*IM, S, 3] of every set, with what their backward needs: the rays K^-1 (u, v, 1), the
    depths, K^-1 per set and the keypoint index of every entry.  Kinv = (K0^-1, K1^-1) replaces torch.linalg.inv(K)."""
    B, N = kps0.shape[0], kps0.shape[2]
    S = sampled.shape[1]
    cell = sampled.long()
    i0, i1 = torch.div(cell, N, rounding_mode="trunc"), cell % N
    bidx = torch.arange(B, device=kps0.device).repeat_interleave(IM).unsqueeze(1).expand(-1, S)
    out = []
    Kis = (torch.linalg.inv(K0), torch.linalg.inv(K1)) if Kinv is None else tuple(k.to(K0.dtype) for k in Kinv)
    for kps, depth, Ki, idx in ((kps0, depth0, Kis[0], i0), (kps1, depth1, Kis[1], i1)):
        Ki = Ki.repeat_interleave(IM, 0)                                                      # [B*IM, 3, 3]
        uv1 = torch.cat([kps[bidx, :2, idx], torch.ones_like(kps[bidx, :1, idx])], -1)       # [B*IM, S, 3]
        ray = uv1 @ Ki.transpose(1, 2)
        z = depth[bidx, 0, idx]
        out.append((z.unsqueeze(-1) * ray, ray, z, Ki, idx))
    return out, bidx


def tail_autograd(kps0, depth0, kps1, depth1, K0, K1, Kori0, Kori1, Rgt, tgt, sampled, inl, p: LossParams):
    """The reference's tail (:140-152, :199-248) composed from the restated helpers, differentiable in the four leaves:
    (loss_value, loss_rot, loss_trans) [B*IM] in the leaves' dtype, or None for the invalid-pose early return."""
    B, IM, IR, S = kps0.shape[0], p.it_matches, p.it_ransac, p.n_sample
    dt, dev = kps0.dtype, kps0.device
    N = kps0.shape[2]
    cell = sampled.long()
    i0, i1 = torch.div(cell, N, rounding_mode="trunc"), cell % N
    bidx = torch.arange(B, device=dev).repeat_interleave(IM).unsqueeze(1).expand(-1, S)
    X = backproject_3d(kps0[bidx, :2, i0], depth0[bidx, :2, i0], K0.repeat_interleave(IM, 0))     # :144-152
    Y = backproject_3d(kps1[bidx, :2, i1], depth1[bidx, :2, i1], K1.repeat_interleave(IM, 0))
    X_v = X.unsqueeze(1).expand(-1, IR, -1, -1).reshape(B * IM * IR, S, 3)
    Y_v = Y.unsqueeze(1).expand(-1, IR, -1, -1).reshape(B * IM * IR, S, 3)
    R, t = weighted_procrustes(X_v, Y_v, inl.to(dt))
    if not (bool(torch.isfinite(R).all()) and bool(torch.isfinite(t).all())):
        return None
    score = soft_inlier_counting_3d(X_v, Y_v, R, t, p.inlier_3d_th).reshape(B * IM, IR)
    rep = IM * IR
    loss_fn = compute_vcre_loss if p.loss_type == "VCRE" else compute_pose_loss
    lv, lr, lt = loss_fn(R, t, Rgt.repeat_interleave(rep, 0), tgt.repeat_interleave(rep, 0), Kori0.repeat_interleave(rep, 0),
                         Kori1.repeat_interleave(rep, 0), vcre_grid(dev).to(dt), p.soft_clipping)
    lv, lr, lt = (x.reshape(B * IM, IR) for x in (lv, lr, lt))
    sm = torch.softmax(score / p.score_temperature, -1)
    loss_rot, loss_trans = (lr * sm).sum(-1), (lt * sm).sum(-1)
    if p.add_null_hypothesis:
        lv = torch.cat([lv, torch.full((B * IM, 1), p.max_loss_null, dtype=dt, device=dev)], -1)
        score = torch.cat([score, torch.full((B * IM, 1), p.th_outliers * S, dtype=dt, device=dev)], -1)
    return (lv * torch.softmax(score / p.score_temperature, -1)).sum(-1), loss_rot, loss_trans


def _skew(y):
    z = torch.zeros_like(y[:, 0])
    return torch.stack([torch.stack([z, -y[:, 2], y[:, 1]], -1), torch.stack([y[:, 2], z, -y[:, 0]], -1),
                        torch.stack([-y[:, 1], y[:, 0], z], -1)], 1)


def procrustes_backward(R, H, G_R, mutation=None):
    """dL/dH of R = V Z U^T (H = U S V^T) from G_R = dL/dR, with no SVD: R H is symmetric at the optimum, so
    P = sym(R H), M = tr(P) I - P, B = G_R R^T, g = (B32 - B23, B13 - B31, B21 - B12) and G_H = -R^T [M^-1 g]x.
    M's eigenvalues are l_j + l_k with the singular values l, the last signed by Z."""
    P = R @ H
    P = (P + P.transpose(1, 2)) / 2
    if mutation == "z_in_m":                              # planted: the unsigned sqrt(H^T H) in place of R H
        _, s, V = torch.svd(H)
        P = V @ torch.diag_embed(s) @ V.transpose(1, 2)
    eye = torch.eye(3, dtype=R.dtype, device=R.device)
    M = P.diagonal(dim1=1, dim2=2).sum(-1)[:, None, None] * eye - P
    Bm = G_R @ R.transpose(1, 2)
    g = torch.stack([Bm[:, 2, 1] - Bm[:, 1, 2], Bm[:, 0, 2] - Bm[:, 2, 0], Bm[:, 1, 0] - Bm[:, 0, 1]], -1)
    y = torch.linalg.solve(M, g)
    G_H = -R.transpose(1, 2) @ _skew(y)
    return -G_H if mutation == "rt_sign" else G_H


def _vcre_backward(R, t, Rgt, tgt, K, grid, g, inverse, mutation=None):
    """G_R, g_t of g * (mean over the grid of one direction's clipped projection distance), vcre_loss's arithmetic,
    and the magnitudes the element bound of tests/loss_tail_check.py charges: max over the grid of
    (1 + (|res0| + |res1|) / |res2|)^2 [n] (the projection's amplification of a relative error in res), and G_R, g_t with every term's absolute value."""
    e = grid.to(R.dtype).unsqueeze(0)                                     # [1, P, 3]
    if inverse:                # res = Rgt R^T (e - t) + Rgt Rgt^T tgt (Rgt, read from fp32, is orthogonal to ~1e-7 only)
        q = e - t.unsqueeze(1)
        tg = tgt.unsqueeze(1) if mutation == "vcre_inverse_tgt" else (tgt.unsqueeze(1) @ Rgt) @ Rgt.transpose(1, 2)
        res = (q @ R) @ Rgt.transpose(1, 2) + tg
    else:                                                                 # res = Rgt^T (R e + t - tgt)
        res = (e @ R.transpose(1, 2) + (t - tgt).unsqueeze(1)) @ Rgt
    x, xg = res @ K.transpose(1, 2), e @ K.transpose(1, 2)
    z = x[..., 2] + 1e-16
    up, ug = x[..., :2] / z.unsqueeze(-1), xg[..., :2] / (xg[..., 2:3] + 1e-16)
    df = ug.clamp(0, 720) - up.clamp(0, 720)
    v = ((df ** 2).sum(-1) + 1e-6).sqrt()
    w = g[:, None] / grid.shape[0]
    gate = ug if mutation == "vcre_gate_gt" else up
    gu = torch.where((gate >= 0) & (gate <= 720), -w.unsqueeze(-1) * df / v.unsqueeze(-1), torch.zeros_like(up))
    gx = torch.stack([gu[..., 0] / z, gu[..., 1] / z, -(gu[..., 0] * x[..., 0] + gu[..., 1] * x[..., 1]) / z ** 2], -1)
    gres = gx @ K
    amp = ((1 + (res[..., 0].abs() + res[..., 1].abs()) / res[..., 2].abs()) ** 2).amax(1)
    # df is a difference of two clipped projections: its error scales with theirs, however small df is
    gua = torch.where((gate >= 0) & (gate <= 720), w.abs().unsqueeze(-1) * (df.abs() + ug.clamp(0, 720) + up.clamp(0, 720))
                      / v.unsqueeze(-1), torch.zeros_like(up))
    gxa = torch.stack([gua[..., 0] / z.abs(), gua[..., 1] / z.abs(),
                       (gua[..., 0] * x[..., 0].abs() + gua[..., 1] * x[..., 1].abs()) / z ** 2], -1)
    gra = gxa @ K.abs()
    if inverse:
        gpp, gppa = gres @ Rgt, gra @ Rgt.abs()
        return (torch.einsum("npi,npj->nij", q, gpp), -(gpp @ R.transpose(1, 2)).sum(1), amp,
                torch.einsum("npi,npj->nij", q.abs(), gppa), (gppa @ R.abs().transpose(1, 2)).sum(1))
    gp, gpa = gres @ Rgt.transpose(1, 2), gra @ Rgt.abs().transpose(1, 2)
    return (torch.einsum("npi,npj->nij", gp, e.expand_as(gp)), gp.sum(1), amp,
            torch.einsum("npi,npj->nij", gpa, e.abs().expand_as(gp)), gpa.sum(1))


def scatter_entries(gP, set_pts, bidx, B, N, IR, absolute=False):
    """Per-(hypothesis, entry) point gradients gP [B*IM*IR, S, 3] of one image, summed over the set's hypotheses, through
    the back-projection X = z K^-1 (u, v, 1) and summed over each keypoint's draws: (dkps [B, 2, N], ddepth [B, 1, N]).
    absolute=True sums |gP| through |K^-1| and |z| (the magnitudes tests/loss_tail_check.py charges rounding on)."""
    _, ray, z, Ki, idx = set_pts
    S = gP.shape[1]
    gP = gP.reshape(-1, IR, S, 3).sum(1)
    if absolute:
        gP, ray, z, Ki = gP.abs(), ray.abs(), z.abs(), Ki.abs()
    g_uv = z.unsqueeze(-1) * (gP @ Ki)[..., :2]
    g_z = (gP * ray).sum(-1)
    dt, dev = gP.dtype, gP.device
    dk = torch.zeros(B, N, 2, dtype=dt, device=dev).index_put_((bidx.reshape(-1), idx.reshape(-1)), g_uv.reshape(-1, 2),
                                                               accumulate=True)
    dd = torch.zeros(B, N, dtype=dt, device=dev).index_put_((bidx.reshape(-1), idx.reshape(-1)), g_z.reshape(-1),
                                                            accumulate=True)
    return dk.transpose(1, 2).contiguous(), dd.unsqueeze(1)


def _last_draw(idx, bidx, B, N):
    """[B*IM, S] bool: the entry that is the last, in the pair's ascending (outer iteration, entry) order, to draw its
    keypoint (the scatter's final addition for that keypoint)."""
    BIM, S = idx.shape
    order = torch.arange(BIM * S, device=idx.device).reshape(BIM, S)
    key = (bidx * N + idx).reshape(-1)
    last = torch.full((B * N,), -1, dtype=torch.long, device=idx.device).scatter_reduce(0, key, order.reshape(-1), "amax")
    return (last[key] == order.reshape(-1)).reshape(BIM, S)


def tail_closed_form(kps0, depth0, kps1, depth1, K0, K1, Kori0, Kori1, Rgt, tgt, sampled, inl, p: LossParams, g_value,
                     g_rot, g_trans, mutation=None, Kinv=None, grid=None):
    """The tail's values and its closed-form backward, the arithmetic csrc/loss_tail.cu runs, in the inputs' dtype.
    Rgt [B, 3, 3], tgt [B, 1, 3]; g_value / g_rot / g_trans [B*IM] are the upstream gradients of loss_value / loss_rot /
    loss_trans.  Kinv = (K0^-1, K1^-1) back-projects in place of torch.linalg.inv (kernel_kinv gives the kernel's);
    grid [196, 3] replaces the fp64 vcre_grid (the kernel reads it in fp32).
    Returns a dict: loss_value, loss_rot, loss_trans [B*IM]; R, t, H, score, G_R, g_t, G_H per hypothesis;
    dkps0, dkps1 [B, 2, N], ddepth0, ddepth1 [B, 1, N]; and under "mag" what tests/loss_tail_check.py's element bound
    needs (per hypothesis: the softmax weights, losses, cosine, M's smallest |eigenvalue|, the VCRE amplification; per
    hypothesis and entry: every gradient term's magnitude).  `mutation` (one of TAIL_MUTATIONS) plants an error."""
    B, N = kps0.shape[0], kps0.shape[2]
    IM, IR, S = p.it_matches, p.it_ransac, p.n_sample
    dt, dev = kps0.dtype, kps0.device
    n = B * IM * IR
    kps0, depth0, kps1, depth1 = (x.detach() for x in (kps0, depth0, kps1, depth1))
    if mutation == "ki_fp64":
        Kinv = None
    sets, bidx = _set_points(kps0, depth0, kps1, depth1, K0, K1, sampled, IM, Kinv)
    (X, *_), (Y, *_) = sets
    Xv, Yv = X.repeat_interleave(IR, 0), Y.repeat_interleave(IR, 0)
    w = inl.to(dt)
    eps = 1e-16
    wn = w / (w.abs().sum(1, keepdim=True) + eps)
    a, b = (wn.unsqueeze(-1) * Xv).sum(1), (wn.unsqueeze(-1) * Yv).sum(1)
    H = (Xv - a.unsqueeze(1)).transpose(1, 2) @ (w.unsqueeze(-1) * (Yv - b.unsqueeze(1)))
    R, _ = weighted_procrustes(Xv, Yv, w)
    t = b - (R @ a.unsqueeze(-1)).squeeze(-1)
    r = Xv @ R.transpose(1, 2) + t.unsqueeze(1) - Yv
    d = ((r ** 2).sum(-1) + 1e-6).sqrt()
    k5 = 5.0 / p.inlier_3d_th
    arg = k5 * (p.inlier_3d_th - d)
    sg = torch.sigmoid(arg.float()).to(dt) if mutation == "sigmoid_fp32" else torch.sigmoid(arg)
    score = sg.sum(1)
    rep = IM * IR
    grid = (vcre_grid(dev) if grid is None else grid).to(dev, dt)
    Rg, tg = Rgt.to(dt).repeat_interleave(rep, 0), tgt.to(dt).reshape(B, 3).repeat_interleave(rep, 0)
    Ko0, Ko1 = Kori0.to(dt).repeat_interleave(rep, 0), Kori1.to(dt).repeat_interleave(rep, 0)
    loss_fn = compute_vcre_loss if p.loss_type == "VCRE" else compute_pose_loss
    lv, lr, lt = loss_fn(R, t.unsqueeze(1), Rg, tg.unsqueeze(1), Ko0, Ko1, grid, p.soft_clipping)
    lv, lr, lt, sc = (x.reshape(B * IM, IR) for x in (lv, lr, lt, score))
    T = p.score_temperature
    sm = torch.softmax(sc / T, -1)
    qn = None
    if p.add_null_hypothesis:
        q = torch.softmax(torch.cat([sc, torch.full((B * IM, 1), p.th_outliers * S, dtype=dt, device=dev)], -1) / T, -1)
        loss_value = (q[:, :IR] * lv).sum(-1) + q[:, IR] * p.max_loss_null
        q, qn = q[:, :IR], q[:, IR]
    else:
        q = sm
        loss_value = (q * lv).sum(-1)
    if mutation == "rot_weights_q":
        sm = q
    loss_rot, loss_trans = (sm * lr).sum(-1), (sm * lt).sum(-1)
    # softmaxes
    gv, gr, gtr = (x.to(dt).reshape(B * IM, 1) for x in (g_value, g_rot, g_trans))
    gs = ((gv * q * (lv - loss_value[:, None]) + gr * sm * (lr - loss_rot[:, None]) + gtr * sm * (lt - loss_trans[:, None]))
          / T).reshape(n)
    gs_mag = ((gv.abs() * q * (lv.abs() + loss_value.abs()[:, None]) + gr.abs() * sm * (lr.abs() + loss_rot.abs()[:, None])
               + gtr.abs() * sm * (lt.abs() + loss_trans.abs()[:, None])) / abs(T)).reshape(n)
    dlv, dlr, dlt = (gv * q).reshape(n), (gr * sm).reshape(n), (gtr * sm).reshape(n)
    dlr_mag, dlt_mag = dlr.abs(), dlt.abs()
    lv, lr = lv.reshape(n), lr.reshape(n)
    G_R = torch.zeros(n, 3, 3, dtype=dt, device=dev)
    g_t = torch.zeros(n, 3, dtype=dt, device=dev)
    G_R_mag, g_t_mag = torch.zeros_like(G_R), torch.zeros_like(g_t)
    vamp = torch.ones(n, dtype=dt, device=dev)
    if p.loss_type == "VCRE":
        graw = dlv * ((1 - lv ** 2) / 80 if p.soft_clipping else 1.0) / 2
        for K, inverse in ((Ko0, False), (Ko1, True)):
            gR_, gt_, amp, gRa, gta = _vcre_backward(R, t, Rg, tg, K, grid, graw, inverse, mutation)
            G_R, g_t = G_R + gR_, g_t + gt_
            G_R_mag, g_t_mag, vamp = G_R_mag + gRa, g_t_mag + gta, torch.maximum(vamp, amp)
    elif p.soft_clipping:
        dlr = dlr + dlv * (1 - torch.tanh(lr / 0.9) ** 2) / 0.9
        dlt = dlt + dlv * (1 - torch.tanh(lt.reshape(n) / 0.9) ** 2) / 0.9
        dlr_mag = dlr_mag + dlv.abs() * (1 - torch.tanh(lr / 0.9) ** 2) / 0.9
        dlt_mag = dlt_mag + dlv.abs() * (1 - torch.tanh(lt.reshape(n) / 0.9) ** 2) / 0.9
    else:
        dlr, dlt = dlr + dlv, dlt + dlv
        dlr_mag, dlt_mag = dlr_mag + dlv.abs(), dlt_mag + dlv.abs()
    # the score through R and t; its direct path through X, Y is added per entry below
    csg = sg * (1 - sg) / d
    g_r = (-k5 * gs)[:, None, None] * csg.unsqueeze(-1) * r
    g_r_mag = (k5 * gs_mag)[:, None, None] * csg.unsqueeze(-1) * r.abs()
    G_R = G_R + torch.einsum("nsi,nsj->nij", g_r, Xv)
    g_t = g_t + g_r.sum(1)
    G_R_mag = G_R_mag + torch.einsum("nsi,nsj->nij", g_r_mag, Xv.abs())
    g_t_mag = g_t_mag + g_r_mag.sum(1)
    # acos(clip(c)): clamp passes the gradient on [-0.99999, 0.99999] only
    c = ((R * Rg).sum((1, 2)) - 1) / 2
    inside = (c >= -ACOS_CLIP) & (c <= ACOS_CLIP)
    if mutation == "acos_edge":
        inside = torch.ones_like(inside)
    cc = c.clamp(-ACOS_CLIP, ACOS_CLIP)
    f = torch.where(inside, dlr * (-1 / (1 - cc ** 2).sqrt()) * 0.5, torch.zeros_like(c))
    f_mag = torch.where(inside, dlr_mag / (1 - cc ** 2).sqrt() * 0.5, torch.zeros_like(c))
    G_R = G_R + f[:, None, None] * Rg
    g_t = g_t + dlt[:, None] * torch.sign(t - tg)
    G_R_mag = G_R_mag + f_mag[:, None, None] * Rg.abs()
    g_t_mag = g_t_mag + dlt_mag[:, None]
    G_R = G_R - g_t.unsqueeze(-1) * a.unsqueeze(1)                       # t = b - R a
    G_R_mag = G_R_mag + g_t_mag.unsqueeze(-1) * a.abs().unsqueeze(1)
    G_H = procrustes_backward(R, H, G_R, mutation)
    # t = b - R a; H's own dependence on the means: sum w_i (Y_i - b) = eps b, sum w_i (X_i - a) = eps a
    g_a = -(R.transpose(1, 2) @ g_t.unsqueeze(-1)).squeeze(-1) - (G_H @ (eps * b).unsqueeze(-1)).squeeze(-1)
    g_b = g_t - (G_H.transpose(1, 2) @ (eps * a).unsqueeze(-1)).squeeze(-1)
    dX = w.unsqueeze(-1) * ((Yv - b.unsqueeze(1)) @ G_H.transpose(1, 2))
    dY = w.unsqueeze(-1) * ((Xv - a.unsqueeze(1)) @ G_H)
    if mutation != "mean_x":
        dX = dX + wn.unsqueeze(-1) * g_a.unsqueeze(1)
    dY = dY + wn.unsqueeze(-1) * g_b.unsqueeze(1)
    if mutation != "score_direct":
        dX = dX + g_r @ R
        dY = dY - g_r
    if mutation == "last_hyp_dropped":
        keep = torch.ones(IR, dtype=dt, device=dev)
        keep[IR - 1] = 0
        keep = keep.repeat(B * IM)[:, None, None]
        dX, dY = dX * keep, dY * keep
    # magnitudes: |G_H| <= |R^T| |[y]x| with |y| <= |g|_2 / lambda_min(M), |g| from |G_R| |R|^T
    P = R @ H
    P = (P + P.transpose(1, 2)) / 2
    M = P.diagonal(dim1=1, dim2=2).sum(-1)[:, None, None] * torch.eye(3, dtype=dt, device=dev) - P
    lam = torch.linalg.eigvalsh(M).abs().amin(-1) if bool(torch.isfinite(M).all()) else torch.zeros(n, dtype=dt, device=dev)
    Bm = G_R_mag @ R.abs().transpose(1, 2)
    g_mag = torch.stack([Bm[:, 2, 1] + Bm[:, 1, 2], Bm[:, 0, 2] + Bm[:, 2, 0], Bm[:, 1, 0] + Bm[:, 0, 1]], -1)
    y_mag = (g_mag.norm(dim=-1) / lam).unsqueeze(-1).expand(-1, 3)
    GH_mag = R.abs().transpose(1, 2) @ _skew(y_mag).abs()
    ga_mag = (R.abs().transpose(1, 2) @ g_t_mag.unsqueeze(-1)).squeeze(-1) + (GH_mag @ (eps * b.abs()).unsqueeze(-1)).squeeze(-1)
    gb_mag = g_t_mag + (GH_mag.transpose(1, 2) @ (eps * a.abs()).unsqueeze(-1)).squeeze(-1)
    TX = (w.unsqueeze(-1) * (((Yv - b.unsqueeze(1)).abs() + b.abs().unsqueeze(1)) @ GH_mag.transpose(1, 2))
          + wn.unsqueeze(-1) * ga_mag.unsqueeze(1) + g_r_mag @ R.abs())
    TY = (w.unsqueeze(-1) * (((Xv - a.unsqueeze(1)).abs() + a.abs().unsqueeze(1)) @ GH_mag)
          + wn.unsqueeze(-1) * gb_mag.unsqueeze(1) + g_r_mag)
    # c r per unit relative pose error: r = R x + t - y carries |x| + |t| + |y| times it, and c = k5 gs sg (1 - sg) / d
    # moves by (k5 + 1 / d) per unit of d
    ell = Xv.abs().sum(-1) + Yv.abs().sum(-1) + t.abs().sum(-1, keepdim=True)
    cres = (k5 * gs_mag)[:, None] * csg * (2 + k5 * d) * ell
    out = {"loss_value": loss_value, "loss_rot": loss_rot, "loss_trans": loss_trans, "R": R, "t": t, "H": H,
           "score": score, "G_R": G_R, "g_t": g_t, "G_H": G_H}
    sens = k5 * (sg * (1 - sg) * (Xv.abs().sum(-1) + Yv.abs().sum(-1) + t.abs().sum(-1, keepdim=True))).sum(1)
    out["mag"] = {"score_sens": sens, "q": q, "qn": qn, "sm": sm, "lv": lv.reshape(B * IM, IR), "lr": lr.reshape(B * IM, IR),
                  "lt": lt.reshape(B * IM, IR), "score": sc, "cos": c, "inside": inside, "lam": lam, "vamp": vamp,
                  "w": w, "X": Xv, "Y": Yv, "a": a, "b": b, "t": t, "TX": TX, "TY": TY, "cres": cres, "sets": sets, "bidx": bidx}
    # back-projection X = z K^-1 (u, v, 1), then the sum over each keypoint's draws
    for name, gP, sp in (("0", dX, sets[0]), ("1", dY, sets[1])):
        if mutation == "scatter_drop_last":
            gP = gP * (~_last_draw(sp[4], bidx, B, N)).to(dt).repeat_interleave(IR, 0).unsqueeze(-1)
        out["dkps" + name], out["ddepth" + name] = scatter_entries(gP, sp, bidx, B, N, IR)
    return out
