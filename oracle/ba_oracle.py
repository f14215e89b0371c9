"""fp64 numpy restatement of ovg_bundle_adjust (csrc/ba.cuh): the same problem, gauge, Levenberg-Marquardt rules, Schur
complement and block-Jacobi PCG, step for step, vectorised over observations.  ``record=True`` also solves every reduced
camera system directly (np.linalg.solve of the dense S) for comparison with the PCG.  The sums run in numpy's order, not the
device's, so results agree to rounding, not bit for bit."""
from __future__ import annotations

import numpy as np

NP = 8                          # per view: rotation increment (3), translation (3), fx, fy
PCG_MAX = 500


def exp_so3(w):
    """Rodrigues' formula for rotation vectors w [..., 3], with its series form below theta^2 = 1e-16."""
    w = np.asarray(w, np.float64)
    th2 = (w * w).sum(-1)
    big = th2 >= 1e-16
    th = np.sqrt(np.where(big, th2, 1.0))
    A = np.where(big, np.sin(th) / th, 1.0)
    B = np.where(big, (1.0 - np.cos(th)) / np.where(big, th2, 1.0), 0.5)
    K = np.zeros(w.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2], K[..., 1, 2] = -w[..., 2], w[..., 1], -w[..., 0]
    K[..., 1, 0], K[..., 2, 0], K[..., 2, 1] = w[..., 2], -w[..., 1], w[..., 0]
    E = B[..., None, None] * (w[..., :, None] * w[..., None, :]) + A[..., None, None] * K
    E += (1.0 - B * th2)[..., None, None] * np.eye(3)
    return E


def reproject(E, K, P, obs):
    """track_reproject per observation: E [m, 3, 4], K [m, 3, 3], P [m, 3], obs [m, 2] -> (X [m, 3], r [m, 2], Z <= 0)."""
    X = ((E[:, :, 0] * P[:, None, 0] + E[:, :, 1] * P[:, None, 1]) + E[:, :, 2] * P[:, None, 2]) + E[:, :, 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[:, 0, 0] * (X[:, 0] / X[:, 2]) + (K[:, 0, 2] + 0.5)
        v = K[:, 1, 1] * (X[:, 1] / X[:, 2]) + (K[:, 1, 2] + 0.5)
    return X, np.stack([u - obs[:, 0], v - obs[:, 1]], 1), X[:, 2] <= 0.0


def jacobians(E, K, P, obs, mask):
    """(residual [m, 2], d r / d camera [m, 2, 8] with the fixed columns zero, d r / d point [m, 2, 3]) for the left rotation
    increment R <- Exp(w) R, t <- t + dt, fx, fy and P <- P + dP."""
    X, r, _ = reproject(E, K, P, obs)
    iz, xn, yn = 1.0 / X[:, 2], X[:, 0] / X[:, 2], X[:, 1] / X[:, 2]
    a = X - E[:, :, 3]
    fxz, fyz = K[:, 0, 0] * iz, K[:, 1, 1] * iz
    z = np.zeros_like(iz)
    jc = np.stack([np.stack([fxz * (-xn * a[:, 1]), fxz * (a[:, 2] + xn * a[:, 0]), fxz * (-a[:, 1]), fxz, z, -fxz * xn, xn, z], 1),
                   np.stack([fyz * (-a[:, 2] - yn * a[:, 1]), fyz * (yn * a[:, 0]), fyz * a[:, 0], z, fyz, -fyz * yn, z, yn], 1)], 1)
    jc = np.where(mask[:, None, :] != 0, jc, 0.0)
    R = E[:, :, :3]
    jp = np.stack([fxz[:, None] * (R[:, 0] - xn[:, None] * R[:, 2]), fyz[:, None] * (R[:, 1] - yn[:, None] * R[:, 2])], 1)
    return r, jc, jp


def inv3_sym(H):
    """Inverse of symmetric 3 x 3 matrices [k, 3, 3] by cofactors, as ba_track_kernel."""
    a, b, c, d, e, f = H[:, 0, 0], H[:, 1, 0], H[:, 2, 0], H[:, 1, 1], H[:, 2, 1], H[:, 2, 2]
    A, B, C = d * f - e * e, c * e - b * f, b * e - c * d
    det = a * A + b * B + c * C
    D, F, E = c * b - a * e, a * d - b * b, a * f - c * c
    out = np.stack([A, B, C, B, E, D, C, D, F], 1).reshape(-1, 3, 3)
    return out / det[:, None, None]


class Problem:
    """The fixed parts of one call: observations, the gauge mask and the refined tracks."""

    def __init__(self, points, offsets, view, obs, ext, intr, refine_focal=True, loss="trivial", loss_scale=1.0):
        self.P0 = np.asarray(points, np.float64).reshape(-1, 3)
        offsets = np.asarray(offsets, np.int64)
        self.view = np.asarray(view, np.int64)
        self.obs = np.asarray(obs, np.float64).reshape(-1, 2)
        ext = np.asarray(ext, np.float32).astype(np.float64)
        intr = np.asarray(intr, np.float32).astype(np.float64)
        self.V, self.n, self.m = ext.shape[0], self.P0.shape[0], self.view.shape[0]
        self.E0, self.K0 = ext.copy(), intr.copy()
        self.track = np.repeat(np.arange(self.n), np.diff(offsets))
        c = ext[0, :, :3].T @ ext[0, :, 3]
        d = ext[1, :, 3] - ext[1, :, :3] @ c
        self.k = int(np.argmax(np.abs(d)))
        mask = np.ones((self.V, NP))
        mask[0, :6] = 0.0
        mask[1, 3 + self.k] = 0.0
        if not refine_focal:
            mask[:, 6:] = 0.0
        self.mask = mask
        self.cauchy, self.c2 = loss == "cauchy", float(loss_scale) ** 2
        _, _, behind = reproject(ext[self.view], intr[self.view], self.P0[self.track], self.obs)
        cnt = np.diff(offsets)
        bad = np.bincount(self.track, behind.astype(np.int64), self.n) > 0
        self.incl = (cnt >= 2) & ~bad
        self.io = self.incl[self.track]                  # refined observations

    def rho(self, s):
        return self.c2 * np.log1p(s / self.c2) if self.cauchy else s

    def weight(self, s):
        return 1.0 / (1.0 + s / self.c2) if self.cauchy else np.ones_like(s)

    def cost(self, E, K, P):
        """(1/2 sum rho over the refined observations, any refined observation at Z <= 0)."""
        io = self.io
        _, r, behind = reproject(E[self.view[io]], K[self.view[io]], P[self.track[io]], self.obs[io])
        return 0.5 * self.rho((r * r).sum(1)).sum(), bool(behind.any())

    def error(self, E, K, P):
        """The mean reprojection distance per track, +inf when some observation has Z <= 0 (tracks' error)."""
        _, r, behind = reproject(E[self.view], K[self.view], P[self.track], self.obs)
        e = np.bincount(self.track, np.sqrt((r * r).sum(1)), self.n) / np.maximum(np.bincount(self.track, minlength=self.n), 1)
        e[np.bincount(self.track, behind.astype(np.int64), self.n) > 0] = np.inf
        return e


def bundle_adjust(points, offsets, view, obs, ext, intr, iterations=100, refine_focal=True, loss="trivial", loss_scale=1.0,
                  record=False):
    """ovg_bundle_adjust restated.  Returns a dict: points [n, 3], extrinsic [V, 3, 4], intrinsic [V, 3, 3], error [n],
    cost [2], steps, accepted, pcg_iterations, status, trace (cost after each step), and with ``record`` a list of
    (PCG solution, direct solution) per solved system."""
    pr = Problem(points, offsets, view, obs, ext, intr, refine_focal, loss, loss_scale)
    V, n, mask = pr.V, pr.n, pr.mask
    E, K, P = pr.E0.copy(), pr.K0.copy(), pr.P0.copy()
    io, vo, to = pr.io, pr.view[pr.io], pr.track[pr.io]
    F, _ = pr.cost(E, K, P)
    res = {"cost0": F, "trace": [], "solves": [], "steps": 0, "accepted": 0, "pcg_iterations": 0, "status": 1}
    mu, nu, lin = 1e4, 2.0, True
    if not io.any():
        res["status"] = 3
        iterations = 0
    while res["steps"] < iterations:
        if lin:
            r, jc, jp = jacobians(E[vo], K[vo], P[to], pr.obs[io], mask[vo])
            w = pr.weight((r * r).sum(1))
            lin = False
        Hp = np.zeros((n, 3, 3))
        np.add.at(Hp, to, w[:, None, None] * np.einsum("ori,orj->oij", jp, jp))
        gp = np.zeros((n, 3))
        np.add.at(gp, to, w[:, None] * np.einsum("ori,or->oi", jp, r))
        U = np.zeros((V, NP, NP))
        np.add.at(U, vo, w[:, None, None] * np.einsum("ori,orj->oij", jc, jc))
        gc = np.zeros((V, NP))
        np.add.at(gc, vo, w[:, None] * np.einsum("ori,or->oi", jc, r))
        if max(np.abs(gp[pr.incl]).max(initial=0.0), np.abs(gc).max()) <= 1e-10:
            res["status"] = 0
            break
        Dp = np.clip(np.diagonal(Hp, axis1=1, axis2=2), 1e-6, 1e32)
        Vinv = np.zeros((n, 3, 3))
        Vinv[pr.incl] = inv3_sym(Hp[pr.incl] + Dp[pr.incl][:, :, None] * np.eye(3) / mu)
        y = np.einsum("pij,pj->pi", Vinv, gp)
        Us = U + np.clip(np.diagonal(U, axis1=1, axis2=2), 1e-6, 1e32)[:, :, None] * np.eye(NP) / mu
        W = w[:, None, None] * np.einsum("ori,ora->oia", jc, jp)             # [m, 8, 3]
        WV = np.einsum("oia,oab->oib", W, Vinv[to])
        Svv = Us.copy()
        np.add.at(Svv, vo, -np.einsum("oib,ojb->oij", WV, W))
        b = -gc.copy()
        np.add.at(b, vo, np.einsum("oia,oa->oi", W, y[to]))
        Lc = np.linalg.cholesky(Svv)

        def precond(rv):
            return np.stack([np.linalg.solve(Lc[v].T, np.linalg.solve(Lc[v], rv[v])) for v in range(V)])

        def apply_s(pv):
            s = np.zeros((n, 3))
            np.add.at(s, to, np.einsum("oia,oi->oa", W, pv[vo]))
            z = np.einsum("pij,pj->pi", Vinv, s)
            q = np.einsum("vij,vj->vi", Us, pv)
            np.add.at(q, vo, -np.einsum("oia,oa->oi", W, z[to]))
            return q

        x = np.zeros((V, NP))
        rr_ = b.copy()
        z = precond(rr_)
        pv = z.copy()
        rz, bb = (rr_ * z).sum(), (b * b).sum()
        tol, rr, it = 1e-10 * np.sqrt(bb), bb, 0
        while it < PCG_MAX and np.sqrt(rr) > tol:
            q = apply_s(pv)
            pq = (pv * q).sum()
            if not pq > 0:
                break
            alpha = rz / pq
            x += alpha * pv
            rr_ -= alpha * q
            rr = (rr_ * rr_).sum()
            it += 1
            if it >= PCG_MAX or not np.sqrt(rr) > tol:
                break
            z = precond(rr_)
            rzn = (rr_ * z).sum()
            pv = z + (rzn / rz) * pv
            rz = rzn
        if record:
            S = np.zeros((V * NP, V * NP))
            for v in range(V):
                S[v * NP:(v + 1) * NP, v * NP:(v + 1) * NP] = Us[v]
            Wd = np.zeros((V * NP, 3 * n))
            for o in range(len(vo)):
                Wd[vo[o] * NP:(vo[o] + 1) * NP, 3 * to[o]:3 * to[o] + 3] += W[o]
            Vd = np.zeros((3 * n, 3 * n))
            for p_ in np.flatnonzero(pr.incl):
                Vd[3 * p_:3 * p_ + 3, 3 * p_:3 * p_ + 3] = Vinv[p_]
            S -= Wd @ Vd @ Wd.T
            res["solves"].append((x.ravel().copy(), np.linalg.solve(S, b.ravel())))
        dc = np.where(mask != 0, x, 0.0)
        s = np.zeros((n, 3))
        np.add.at(s, to, np.einsum("oia,oi->oa", W, dc[vo]))
        dp = np.einsum("pij,pj->pi", Vinv, -gp - s)
        dp[~pr.incl] = 0.0
        # trial
        En, Kn = E.copy(), K.copy()
        rot = mask[:, 0] != 0
        En[rot, :, :3] = np.einsum("vij,vjk->vik", exp_so3(dc[rot, :3]), E[rot, :, :3])
        En[:, :, 3] = np.where(mask[:, 3:6] != 0, E[:, :, 3] + dc[:, 3:6], E[:, :, 3])
        Kn[:, 0, 0] = np.where(mask[:, 6] != 0, K[:, 0, 0] + dc[:, 6], K[:, 0, 0])
        Kn[:, 1, 1] = np.where(mask[:, 7] != 0, K[:, 1, 1] + dc[:, 7], K[:, 1, 1])
        Pn = P + dp
        free_x = np.concatenate([E[:, :, 3][mask[:, 3:6] != 0], K[:, 0, 0][mask[:, 6] != 0], K[:, 1, 1][mask[:, 7] != 0]])
        step = np.sqrt((dc * dc).sum() + (dp * dp).sum())
        xnorm = np.sqrt((free_x * free_x).sum() + (P[pr.incl] ** 2).sum())
        res["steps"] += 1
        res["pcg_iterations"] += it
        if step <= 1e-8 * (xnorm + 1e-8):
            res["status"] = 0
            res["trace"].append(F)
            break
        Fn, behind = pr.cost(En, Kn, Pn)
        jd = np.einsum("ori,oi->or", jc, dc[vo]) + np.einsum("ora,oa->or", jp, dp[to])
        model = (w * (-(r * jd).sum(1) - 0.5 * (jd * jd).sum(1))).sum()
        with np.errstate(divide="ignore", invalid="ignore"):
            rho = (F - Fn) / model
        stop = False
        if not behind and np.isfinite(Fn) and model > 0 and rho > 1e-3:
            qq = 2.0 * rho - 1.0
            mu = mu / max(1.0 / 3.0, 1.0 - qq * qq * qq)
            nu = 2.0
            stop = F - Fn <= 1e-6 * F
            F, E, K, P, lin = Fn, En, Kn, Pn, True
            res["accepted"] += 1
        else:
            mu, nu = mu / nu, 2.0 * nu
            if mu < 1e-32:
                res["status"] = 2
                stop = True
        res["trace"].append(F)
        if stop:
            if res["status"] == 1:
                res["status"] = 0
            break
    res.update(points=P, extrinsic=E, intrinsic=K, error=pr.error(E, K, P), cost=np.array([res.pop("cost0"), F]),
               problem=pr)
    return res
