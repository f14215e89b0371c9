"""fp64 numpy / scipy statement of scene.evaluate's definitions (include/ovg.h, INTEGRATION.md "Evaluation"), written from those
definitions and evo's documented formulas: APE (translation part) and RPE (delta 1, all pairs) after the Umeyama Sim(3) of the
camera centres, the pairwise AUC / RRA / RTA protocol of the VGGT family, median-scaled depth errors, and point-map accuracy,
completeness and normal consistency by cKDTree."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

TAUS = (5, 10, 30)


def camera_ok(ext, intr):
    """[S] bool: fx, fy > 0 and the world-to-camera extrinsic [S, 3, 4] finite."""
    ext, intr = np.asarray(ext), np.asarray(intr)
    return (intr[:, 0, 0] > 0) & (intr[:, 1, 1] > 0) & np.isfinite(ext[:, :3, :4]).all(axis=(1, 2))


def cam_to_world(ext):
    """(R^T [n, 3, 3], c = -R^T t [n, 3]) in fp64 of world-to-camera [n, 3, 4]."""
    e = np.asarray(ext, np.float64)
    Rt = np.swapaxes(e[:, :3, :3], 1, 2)
    return Rt, -np.einsum("nij,nj->ni", Rt, e[:, :3, 3])


def angle(R):
    """Rotation angle in degrees of R [..., 3, 3]: atan2(|(R32 - R23, R13 - R31, R21 - R12)| / 2, (tr R - 1) / 2)."""
    v = np.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
    return np.degrees(np.arctan2(np.linalg.norm(v, axis=-1) / 2, (np.trace(R, axis1=-2, axis2=-1) - 1) / 2))


def umeyama(src, dst):
    """(A = c R [3, 3], t [3], c, RMS residual) mapping src onto dst [n, 3] (Umeyama 1991, eqs. 40-42); ValueError when n < 3
    or the points are collinear."""
    s, d = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    n = len(s)
    if n < 3:
        raise ValueError("fewer than 3 points")
    ms, md = s.mean(0), d.mean(0)
    es, ed = s - ms, d - md
    var = (es ** 2).sum() / n
    U, D, Vt = np.linalg.svd(ed.T @ es / n)
    if var == 0 or not D[1] > 1e-12 * D[0]:
        raise ValueError("collinear or coincident points")
    S = np.diag([1.0, 1.0, -1.0 if np.linalg.det(U) * np.linalg.det(Vt) < 0 else 1.0])
    c = np.trace(np.diag(D) @ S) / var
    A = c * U @ S @ Vt
    t = md - A @ ms
    r = d - (s @ A.T + t)
    return A, t, c, float(np.sqrt((r ** 2).sum(1).mean()))


def centres_ok(ext):
    """[S] bool: the camera centre -R^T t of world-to-camera ext [S, 3, 4], rounded to fp32, is finite."""
    with np.errstate(all="ignore"):
        return np.isfinite(cam_to_world(ext)[1].astype(np.float32)).all(1)


def pose_metrics(gt_ext, gt_intr, pred_ext, views=None, sim3=None, chunk=None):
    """The pose group over ``views`` (default all, ascending) with a ground-truth camera and a finite prediction whose fp32
    centres are both finite.  ``sim3`` (fp64 [4, 4]) replaces the oracle's own Umeyama fit in the RPE, to check the later
    stages given the device's fit.  ``chunk``: pairs per step of ``pair_errors``, to bound memory at many views."""
    gt_ext, pred_ext = np.asarray(gt_ext, np.float32)[:, :3, :4], np.asarray(pred_ext, np.float32)[:, :3, :4]
    S = len(gt_ext)
    views = sorted(range(S) if views is None else views)
    ok = camera_ok(gt_ext, gt_intr) & np.isfinite(pred_ext).all(axis=(1, 2))
    ok &= centres_ok(gt_ext) & centres_ok(pred_ext)
    idx = np.array([v for v in views if ok[v]], dtype=np.int64)
    n = len(idx)
    Rg, cg = cam_to_world(gt_ext[idx])
    Rp, cp = cam_to_world(pred_ext[idx])
    # the fit sees the centres rounded once to fp32
    A, t, c, ate = umeyama(cp.astype(np.float32), cg.astype(np.float32))
    fit = np.eye(4)
    fit[:3, :3], fit[:3, 3] = A, t
    if sim3 is not None:
        fit = np.asarray(sim3, np.float64)
    A, t = fit[:3, :3], fit[:3, 3]
    s = np.linalg.norm(A[:, 0])
    Ra = A / s
    Rpa = Ra @ Rp                                   # R_a R (camera-to-world rotations)
    cpa = cp @ A.T + t                              # s R_a c + t_a
    rpe = rpe_errors(Rg, cg, Rpa, cpa)
    pairs, rre, rte = pair_errors(gt_ext[idx], pred_ext[idx], chunk)
    out = {"n": n, "views": idx, "sim3": fit, "ate": ate, "rpe": rpe,
           "rpe_trans": float(np.sqrt((rpe[:, 0] ** 2).mean())) if n >= 2 else np.nan,
           "rpe_rot": float(np.sqrt((rpe[:, 1] ** 2).mean())) if n >= 2 else np.nan,
           "pairs": idx[pairs], "pair_errors": np.stack([rre, rte], -1)}
    out.update(pair_scores(rre, rte))
    return out


def rpe_errors(Rq, cq, Rp, cp):
    """[n - 1, 2] = |t(E)|, angle(R(E)) of E = (Q_k^-1 Q_k+1)^-1 (P_k^-1 P_k+1), poses camera-to-world (R, c)."""
    def rel(R, c):
        return np.einsum("nji,njk->nik", R[:-1], R[1:]), np.einsum("nji,nj->ni", R[:-1], c[1:] - c[:-1])
    Rgr, tgr = rel(Rq, cq)
    Rpr, tpr = rel(Rp, cp)
    RE = np.einsum("nji,njk->nik", Rgr, Rpr)
    tE = np.einsum("nji,nj->ni", Rgr, tpr - tgr)
    return np.stack([np.linalg.norm(tE, axis=-1), angle(RE)], -1).reshape(-1, 2)


def pair_errors(gt_ext, pred_ext, chunk=None):
    """(pairs [P, 2] of positions i < j, RRE [P], RTE [P]) in degrees; relative poses R_ij = R_j R_i^T, t_ij = t_j - R_ij t_i.
    ``chunk``: at most that many pairs per step (each pair's values are computed on their own either way)."""
    n = len(gt_ext)
    ii, jj = np.triu_indices(n, 1)
    gt, pred = np.asarray(gt_ext, np.float64), np.asarray(pred_ext, np.float64)
    step = max(len(ii), 1) if chunk is None else int(chunk)
    rre, rte = np.empty(len(ii)), np.empty(len(ii))
    for a in range(0, len(ii), step):
        i, j = ii[a:a + step], jj[a:a + step]
        rel = []
        for e in (gt, pred):
            R, t = e[:, :3, :3], e[:, :3, 3]
            Rij = R[j] @ np.swapaxes(R[i], 1, 2)
            rel.append((Rij, t[j] - np.einsum("pij,pj->pi", Rij, t[i])))
        (Rg, tg), (Rp, tp) = rel
        rre[a:a + step] = angle(np.swapaxes(Rg, 1, 2) @ Rp)
        ng, np_ = np.linalg.norm(tg, axis=-1), np.linalg.norm(tp, axis=-1)
        e = np.degrees(np.arctan2(np.linalg.norm(np.cross(tg, tp), axis=-1), (tg * tp).sum(-1)))
        rte[a:a + step] = np.where((ng > 0) & (np_ > 0), np.minimum(e, 180.0 - e), 90.0)
    return np.stack([ii, jj], -1), rre, rte


def pair_scores(rre, rte):
    """auc / rra / rta fp64 [3] at TAUS: numpy's mean(cumsum(histogram(err, arange(tau + 1))[0]) / P), (rre < tau).mean()."""
    err = np.maximum(rre, rte)
    P = len(err)
    if P == 0:
        return {k: np.full(3, np.nan) for k in ("auc", "rra", "rta")}
    auc = [np.mean(np.cumsum(np.histogram(err, bins=np.arange(tau + 1))[0]) / P) for tau in TAUS]
    return {"auc": np.array(auc), "rra": np.array([(rre < tau).mean() for tau in TAUS]),
            "rta": np.array([(rte < tau).mean() for tau in TAUS])}


def depth_valid(gt, pred, mask=None, views=None):
    """[S, ...] bool: the view is scored, the mask set, g > 0 and g, p finite."""
    gt, pred = np.asarray(gt, np.float32), np.asarray(pred, np.float32)
    ok = (gt > 0) & np.isfinite(gt) & np.isfinite(pred)
    if mask is not None:
        ok &= np.asarray(mask) != 0
    if views is not None:
        sel = np.zeros(len(gt), bool)
        sel[list(views)] = True
        ok &= sel.reshape((-1,) + (1,) * (gt.ndim - 1))
    return ok


def depth_metrics(gt, pred, mask=None, views=None, chunk=None):
    """The depth group of gt, pred fp32 [S, H, W] after per-scene median scaling, in fp64; per view too.  ``chunk``: the fp64
    per-pixel terms of that many views at a time, summed view by view, to bound memory at many pixels."""
    gt, pred = np.asarray(gt, np.float32), np.asarray(pred, np.float32)
    ok = depth_valid(gt, pred, mask, views)
    S = len(gt)
    out = {"pixels": int(ok.sum())}
    if not ok.any():
        nan = np.nan
        out.update(scale=nan, median_gt=nan, median_pred=nan, abs_rel=nan, sq_rel=nan, rmse=nan, delta=np.full(3, nan),
                   delta_counts=np.zeros(3, np.int64), view_abs_rel=np.full(S, nan), view_delta1=np.full(S, nan),
                   view_pixels=np.zeros(S, np.int64))
        return out
    mg, mp = np.percentile(gt[ok], 50), np.percentile(pred[ok], 50)
    s = np.float64(mg) / np.float64(mp)
    if chunk is not None:
        return _depth_chunked(gt, pred, ok, s, mg, mp, int(chunk), out)
    g = gt.astype(np.float64)
    sp = s * pred.astype(np.float64)
    with np.errstate(all="ignore"):
        e = sp - g
        are, sre, se = np.abs(e) / g, e * e / g, e * e
        r = np.maximum(sp / g, g / sp)
    d = [(r < 1.25 ** k) & ok for k in (1, 2, 3)]
    n = ok.sum()
    out.update(scale=s, median_gt=mg, median_pred=mp, abs_rel=are[ok].sum() / n, sq_rel=sre[ok].sum() / n,
               rmse=np.sqrt(se[ok].sum() / n), delta_counts=np.array([x.sum() for x in d]),
               delta=np.array([x.sum() / n for x in d]))
    vp = ok.reshape(S, -1).sum(1)
    with np.errstate(all="ignore"):
        out["view_abs_rel"] = np.where(ok, are, 0).reshape(S, -1).sum(1) / np.where(vp > 0, vp, np.nan)
        out["view_delta1"] = d[0].reshape(S, -1).sum(1) / np.where(vp > 0, vp, np.nan)
    out["view_pixels"] = vp
    return out


def _depth_chunked(gt, pred, ok, s, mg, mp, chunk, out):
    """depth_metrics' sums per view, ``chunk`` views at a time, then over the views in order."""
    S = len(gt)
    tot = np.zeros((S, 7))                                   # sum |e| / g, sum e^2 / g, sum e^2, pixels, delta counts (3)
    for a in range(0, S, chunk):
        k = ok[a:a + chunk].reshape(min(chunk, S - a), -1)
        g = gt[a:a + chunk].reshape(k.shape).astype(np.float64)
        sp = s * pred[a:a + chunk].reshape(k.shape).astype(np.float64)
        with np.errstate(all="ignore"):
            e = sp - g
            r = np.maximum(sp / g, g / sp)
            terms = [np.abs(e) / g, e * e / g, e * e]
        tot[a:a + chunk, :3] = np.stack([np.where(k, t, 0).sum(1) for t in terms], 1)
        tot[a:a + chunk, 3] = k.sum(1)
        tot[a:a + chunk, 4:] = np.stack([((r < 1.25 ** q) & k).sum(1) for q in (1, 2, 3)], 1)
    n = tot[:, 3].sum()
    vp = tot[:, 3].astype(np.int64)
    counts = tot[:, 4:].sum(0).astype(np.int64)
    out.update(scale=s, median_gt=mg, median_pred=mp, abs_rel=tot[:, 0].sum() / n, sq_rel=tot[:, 1].sum() / n,
               rmse=np.sqrt(tot[:, 2].sum() / n), delta_counts=counts, delta=counts / n)
    with np.errstate(all="ignore"):
        out["view_abs_rel"] = tot[:, 0] / np.where(vp > 0, vp, np.nan)
        out["view_delta1"] = tot[:, 4] / np.where(vp > 0, vp, np.nan)
    out["view_pixels"] = vp
    return out


def unproject(depth, ext, intr):
    """World points fp64 [S, H, W, 3] of depth [S, H, W] through world-to-camera ext [S, 3, 4] and intr [S, 3, 3]."""
    d = np.asarray(depth, np.float64)
    S, H, W = d.shape
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    K = np.asarray(intr, np.float64)
    x = (u - K[:, 0, 2, None, None]) * d / K[:, 0, 0, None, None]
    y = (v - K[:, 1, 2, None, None]) * d / K[:, 1, 1, None, None]
    cam = np.stack([x, y, d], -1)
    Rt, c = cam_to_world(ext)
    return np.einsum("sij,shwj->shwi", Rt, cam) + c[:, None, None, :]


def sim3_apply(sim3, pts):
    """ovg_sim3_apply's documented rounding of fp32 points [..., 3]: ((A_r0 x + A_r1 y) + A_r2 z) + t_r in fp64, rounded once."""
    A, t = np.asarray(sim3, np.float64)[:3, :3], np.asarray(sim3, np.float64)[:3, 3]
    p = np.asarray(pts, np.float32).astype(np.float64)
    out = [((A[r, 0] * p[..., 0] + A[r, 1] * p[..., 1]) + A[r, 2] * p[..., 2]) + t[r] for r in range(3)]
    return np.stack(out, -1).astype(np.float32)


def grid_normals(points, keep):
    """Normals fp64 [S, H, W, 3] (NaN where none) of points [S, H, W, 3] over keep [S, H, W]: normalize((P[x+1] - P[x-1]) x
    (P[y+1] - P[y-1])) where the pixel and its four neighbours are kept and the cross product is not zero."""
    P = np.asarray(points, np.float32).astype(np.float64)
    k = np.asarray(keep, bool)
    S, H, W = k.shape
    out = np.full((S, H, W, 3), np.nan)
    inner = np.zeros_like(k)
    inner[:, 1:-1, 1:-1] = k[:, 1:-1, 1:-1] & k[:, 1:-1, 2:] & k[:, 1:-1, :-2] & k[:, 2:, 1:-1] & k[:, :-2, 1:-1]
    a = np.zeros_like(P)
    b = np.zeros_like(P)
    a[:, :, 1:-1] = P[:, :, 2:] - P[:, :, :-2]
    b[:, 1:-1] = P[:, 2:] - P[:, :-2]
    c = np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                  a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)
    ln = np.sqrt((c[..., 0] * c[..., 0] + c[..., 1] * c[..., 1]) + c[..., 2] * c[..., 2])
    has = inner & (ln > 0)
    out[has] = c[has] / ln[has][:, None]
    return out


def nearest(queries, data):
    """(distance fp64, index) of each query's nearest data point, by cKDTree in fp64."""
    d, i = cKDTree(np.asarray(data, np.float64)).query(np.asarray(queries, np.float64), k=1)
    return d, i


def point_metrics(pred_aligned, gt_points, keep):
    """The point group's distances and normal consistency between the aligned prediction and the ground truth [S, H, W, 3]
    (fp32 values) over the shared pixel set keep [S, H, W]."""
    k = np.asarray(keep, bool)
    P, G = np.asarray(pred_aligned, np.float32), np.asarray(gt_points, np.float32)
    p, g = P[k], G[k]
    npn, ngn = grid_normals(P, k)[k], grid_normals(G, k)[k]
    acc, ia = nearest(p, g)
    comp, ic = nearest(g, p)

    def nc(na, nb):
        both = ~np.isnan(na[:, 0]) & ~np.isnan(nb[:, 0])
        return np.abs((na[both] * nb[both]).sum(-1)).mean() if both.any() else np.nan
    nca, ncc = nc(npn, ngn[ia]), nc(ngn, npn[ic])
    return {"pixels": int(k.sum()), "acc_dist": acc, "comp_dist": comp, "acc": acc.mean(), "comp": comp.mean(),
            "acc_median": np.percentile(acc.astype(np.float32), 50), "comp_median": np.percentile(comp.astype(np.float32), 50),
            "chamfer": (acc.mean() + comp.mean()) / 2, "nc_acc": nca, "nc_comp": ncc, "nc": (nca + ncc) / 2}
