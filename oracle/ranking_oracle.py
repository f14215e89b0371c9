"""Image ranking restated (datasets/utils/image_ranking.py:9-140, compute_ranking) in numpy; it does not read the reference.

- `dtypes`: the reference's output and compute dtypes for an input dtype, N and path.
- `operands` / `truth`: the fp64 distances in the device kernel's operation order (ovg_compute_ranking): the fp64 mean of
  |t| in the kernel's fixed reduction order, elementwise products and sums with no matmul (numpy neither fuses nor
  reorders them), np.arccos in place of the device's acos.
- `bound`: a per-entry bound on the reference's own error against that truth: the trace and cosine perturbed by
  delta = 8 eps of the reference's compute dtype and pushed through arccos, delta relative on the translation term and on
  the magnitudes of t_i and t_j (the reference normalizes and subtracts in its own dtype), and delta relative on the sum.
- `isolated` / `ranking_agrees`: the positions of a ranking that the reference's error cannot reorder.
- `reference_numpy`: the reference's path restated for timing ([N, N, 3, 3] matmul up to 6000 views, fp32 blocks above).
"""
from __future__ import annotations

import numpy as np

CHUNKED_ABOVE = 6000          # the batched path's switch to fp32 blocks
PREP_THREADS = 256            # rank_prep_kernel's reduction width
DEG = 180.0 / np.pi


def dtypes(in_dtype, N: int, batched: bool = True, chunked: bool = False):
    """(dists dtype, compute dtype) of the reference: chunked (forced, or batched above 6000 views) -> fp32 / fp32; batched
    -> input / input; the per-pair loop -> fp64 / input."""
    in_dtype = np.dtype(in_dtype)
    if chunked or (batched and N > CHUNKED_ABOVE):
        return np.dtype(np.float32), np.dtype(np.float32)
    return (in_dtype if batched else np.dtype(np.float64)), in_dtype


def kernel_lambda(lambda_t: float, compute) -> float:
    """lambda_t as the reference applies it: a Python float times an fp32 array stays fp32 in numpy."""
    return float(np.float32(lambda_t)) if np.dtype(compute) == np.float32 else float(lambda_t)


def mean_norm(t: np.ndarray) -> float:
    """The kernel's mean of |t| (fp64): thread k sums views k, k + 256, ... in order, then a tree over the 256 partials."""
    x, y, z = (t[:, c].astype(np.float64) for c in range(3))
    nrm = np.sqrt((x * x + y * y) + z * z)
    rows = -(-len(nrm) // PREP_THREADS)
    pad = np.zeros(rows * PREP_THREADS)
    pad[:len(nrm)] = nrm
    acc = np.zeros(PREP_THREADS)
    for r in range(rows):
        acc = acc + pad[r * PREP_THREADS:(r + 1) * PREP_THREADS]
    h = PREP_THREADS // 2
    while h:
        acc[:h] = acc[:h] + acc[h:2 * h]
        h //= 2
    return acc[0] / len(nrm)


def operands(E, normalize: bool, out_dtype):
    """R [N, 3, 3] and t [N, 3] in fp64 as the kernel packs them: t / mean |t| rounded to the input dtype, then everything
    rounded to fp32 when the output is fp32."""
    E = np.asarray(E)
    R = E[:, :3, :3].astype(np.float64)
    t = E[:, :3, 3].astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        if normalize:
            t = (t / mean_norm(t)).astype(E.dtype).astype(np.float64)
    if np.dtype(out_dtype) == np.float32:
        R = R.astype(np.float32).astype(np.float64)
        t = t.astype(np.float32).astype(np.float64)
    return R, t


def truth(E, lambda_t: float = 1.0, normalize: bool = True, batched: bool = True, chunked: bool = False, rows=None):
    """fp64 distances of rows (all by default) in the kernel's operation order.  Returns a dict: d [n, N] fp64, its two
    terms rot and trans, the v = (trace - 1) / 2 before the clip, absp = the sum of |products| of the trace, the norms
    of t_i and t_j, the dists and compute dtypes, and lambda as applied."""
    E = np.asarray(E)
    N = E.shape[0]
    out, comp = dtypes(E.dtype, N, batched, chunked)
    lam = kernel_lambda(lambda_t, comp)
    R, t = operands(E, normalize, out)
    rows = np.arange(N) if rows is None else np.asarray(rows)
    Ri, ti = R[rows][:, None], t[rows][:, None]
    Rj, tj = R[None], t[None]
    with np.errstate(invalid="ignore", over="ignore"):
        p = Ri * Rj                                                    # [n, N, 3, 3]: R_i[k, c] R_j[k, c]
        m = (p[..., 0, :] + p[..., 1, :]) + p[..., 2, :]               # diagonal of R_i^T R_j, summed over k in order
        tr = (m[..., 0] + m[..., 1]) + m[..., 2]
        v = (tr - 1.0) * 0.5
        rot = (np.arccos(np.clip(v, -1.0, 1.0)) * DEG) / 180.0
        dt = ti - tj
        tn = np.sqrt((dt[..., 0] * dt[..., 0] + dt[..., 1] * dt[..., 1]) + dt[..., 2] * dt[..., 2])
        trans = lam * tn
        d = rot + trans
        absp = np.abs(p).sum(axis=(-1, -2))
        ni = np.sqrt((ti * ti).sum(-1))
        nj = np.sqrt((tj * tj).sum(-1))
    return dict(d=d, rot=rot, trans=trans, tn=tn, v=v, absp=absp, ni=ni, nj=nj, out=out, compute=comp, lam=lam)


def bound(tr: dict) -> np.ndarray:
    """Per-entry bound on |reference - truth| (see the module docstring)."""
    delta = 8 * np.finfo(tr["compute"]).eps
    with np.errstate(invalid="ignore", over="ignore"):
        dv = delta * (tr["absp"] + 1.0)
        lo = np.arccos(np.clip(tr["v"] + dv, -1.0, 1.0)) / np.pi
        hi = np.arccos(np.clip(tr["v"] - dv, -1.0, 1.0)) / np.pi
        b_rot = np.maximum(hi - tr["rot"], tr["rot"] - lo) + delta * tr["rot"]
        b_trans = delta * abs(tr["lam"]) * (tr["tn"] + tr["ni"] + tr["nj"])
        return b_rot + b_trans + delta * np.abs(tr["d"])


def isolated(d, rank, b) -> np.ndarray:
    """bool [n, N]: position p of each row (in rank's order of d) is farther than the two bounds from both neighbours, so
    no error within the bounds can move it.  NaN sorts last, as +inf; two NaNs or infs are never apart."""
    s = np.take_along_axis(np.asarray(d, np.float64), rank, axis=1)
    bs = np.nan_to_num(np.take_along_axis(b, rank, axis=1), nan=0.0)
    s = np.where(np.isnan(s), np.inf, s)
    with np.errstate(invalid="ignore"):
        sep = (s[:, 1:] - s[:, :-1]) > (bs[:, 1:] + bs[:, :-1])
    edge = np.ones((s.shape[0], 1), bool)
    return np.concatenate([edge, sep], 1) & np.concatenate([sep, edge], 1)


def ranking_agrees(ref_d, ref_rank, b, other_rank) -> np.ndarray:
    """bool [n, N]: other_rank equals the reference's ranking at every position isolated in the reference's distances."""
    iso = isolated(ref_d, ref_rank, b)
    return ~iso | (np.asarray(other_rank) == ref_rank)


def within_ulps(got, tr: dict, ulps: int = 4) -> np.ndarray:
    """bool [n, N]: got lies within `ulps` ulp of the dists dtype (of the larger of the two terms) of the truth rounded to
    that dtype; NaN where the truth is NaN."""
    out = tr["out"]
    want = tr["d"].astype(out)
    got = np.asarray(got)
    with np.errstate(invalid="ignore", over="ignore"):
        scale = np.maximum(np.abs(tr["rot"]), np.abs(tr["trans"])).astype(out)
        tol = ulps * np.spacing(np.where(np.isfinite(scale), scale, 0).astype(out)).astype(np.float64)
        close = np.abs(got.astype(np.float64) - want.astype(np.float64)) <= tol
    return close | (got == want) | (np.isnan(got) & np.isnan(want))


def reference_numpy(E, lambda_t: float = 1.0, normalize: bool = True, batched: bool = True, chunk=None):
    """The reference's host computation restated for timing: [N, N, 3, 3] products up to 6000 views, fp32 blocks of 1000
    views above (or of `chunk` views at any N), then argsort.  Returns (ranking int64, dists)."""
    E = np.array(E, copy=True)
    if normalize:
        t = E[:, :3, 3]
        E[:, :3, 3] = t / np.mean(np.linalg.norm(t, axis=1))
    N = len(E)
    block = chunk or 1000
    if batched and N <= CHUNKED_ABOVE and chunk is None:
        R, t = E[:, :3, :3], E[:, :3, 3]
        M = np.swapaxes(R, 1, 2)[:, None] @ R[None]
        c = np.clip((np.trace(M, axis1=2, axis2=3) - 1) / 2, -1.0, 1.0)
        dists = np.degrees(np.arccos(c)) / 180.0 + lambda_t * np.linalg.norm(t[:, None] - t[None], axis=2)
    elif batched:
        R, t = E[:, :3, :3].astype(np.float32), E[:, :3, 3].astype(np.float32)
        Rt = np.swapaxes(R, 1, 2)
        dists = np.empty((N, N), np.float32)
        for a in range(0, N, block):
            for b in range(0, N, block):
                M = Rt[a:a + block, None] @ R[None, b:b + block]
                c = np.clip((np.trace(M, axis1=2, axis2=3) - 1) / 2, -1.0, 1.0)
                rot = (np.degrees(np.arccos(c)) / 180.0).astype(np.float32)
                dists[a:a + block, b:b + block] = rot + lambda_t * np.linalg.norm(t[a:a + block, None] - t[None, b:b + block],
                                                                                  axis=2)
    else:
        raise NotImplementedError("the per-pair loop is not restated")
    return np.argsort(dists, axis=1), dists
