"""numpy fp64 restatement of OmniVGGT.reconstruct  --  TEST INFRASTRUCTURE (see oracle/omnivggt_oracle.py).

The chunk schedule, the Umeyama (1991) similarity with the library's degeneracy rules, the keep masks, the fp64-once
application of a Sim(3) to a chunk's outputs, and the merge.  The reference has no long-capture code, so nothing here is
pinned to reference outputs: tests/test_long_capture.py pins the estimate to planted transforms and its rotation to
scipy's Rotation.align_vectors, and the libovg kernels to these functions.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

STATUS_OK, STATUS_FEW, STATUS_SIGMA, STATUS_RANK = 0, 1, 2, 3


def schedule(S: int, chunk: int, overlap: int) -> List[Tuple[int, int]]:
    """(start, end) of every chunk: one chunk when S <= chunk; else starts 0, step, 2 step, ... (step = chunk - overlap) while
    start + chunk < S, then a last chunk at S - chunk.  Every chunk has chunk views."""
    if S <= chunk:
        return [(0, S)]
    step = chunk - overlap
    out = []
    start = 0
    while start + chunk < S:
        out.append((start, start + chunk))
        start += step
    out.append((S - chunk, S))
    return out


def new_views(chunks: Sequence[Tuple[int, int]]) -> List[Tuple[int, int]]:
    """The views each chunk adds to the merge: [end of the previous chunk, end), all of chunk 0."""
    return [(a if k == 0 else chunks[k - 1][1], b) for k, (a, b) in enumerate(chunks)]


def reindex(idx: Optional[Sequence[int]], start: int, end: int) -> List[int]:
    """A chunk's members of a list of global view indices, as indices into the chunk."""
    return [int(i) - start for i in (idx or []) if start <= int(i) < end]


def umeyama(src: np.ndarray, dst: np.ndarray, keep: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(sim3 fp64 [4, 4], stats fp64 [4] = kept count, status, RMS residual, c): Umeyama eqs. 40-42 with uniform weights over
    the kept pairs with finite coordinates; the identity (c = 1) with a non-zero status for fewer than 3 pairs (1),
    sigma^2 == 0 (2), or a second singular value not above 1e-12 times the first (3)."""
    s = np.asarray(src, np.float64).reshape(-1, 3)
    d = np.asarray(dst, np.float64).reshape(-1, 3)
    k = np.isfinite(s).all(1) & np.isfinite(d).all(1)
    if keep is not None:
        k &= np.asarray(keep).reshape(-1) != 0
    s, d = s[k], d[k]
    n = len(s)
    sim3, c, status = np.eye(4), 1.0, STATUS_OK
    if n < 3:
        status = STATUS_FEW
    else:
        ms, md = s.mean(0), d.mean(0)
        es, ed = s - ms, d - md
        var = (es * es).sum() / n
        if var == 0.0:
            status = STATUS_SIGMA
        else:
            U, D, Vt = np.linalg.svd(ed.T @ es / n)
            if not D[1] > 1e-12 * D[0]:
                status = STATUS_RANK
            else:
                S = np.diag([1.0, 1.0, -1.0 if np.linalg.det(U) * np.linalg.det(Vt) < 0 else 1.0])
                R = U @ S @ Vt
                c = float(np.trace(np.diag(D) @ S) / var)
                sim3[:3, :3] = c * R
                sim3[:3, 3] = md - c * R @ ms
    rms = float(np.sqrt(((d - (s @ sim3[:3, :3].T + sim3[:3, 3])) ** 2).sum() / n)) if n else 0.0
    return sim3, np.array([n, status, rms, c], np.float64)


def keep_mask(conf: np.ndarray, conf_percent: float, floor: float = 1e-5, threshold: Optional[float] = None) -> np.ndarray:
    """point_cloud's rule: conf >= percentile(conf, conf_percent) and conf > floor (threshold: a given fp32 threshold)."""
    c = np.asarray(conf, np.float32)
    thr = np.percentile(c, conf_percent) if threshold is None else np.float32(threshold)
    return (c >= thr) & (c > floor)


def _dot3(a0, a1, a2, b0, b1, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def apply(sim3: np.ndarray, points=None, depth=None, ext=None, dtype=np.float32) -> Dict[str, np.ndarray]:
    """sim3 [[A, t], [0, 1]] applied as ovg_sim3_apply does: c = sqrt((A00^2 + A10^2) + A20^2), R = A / c; each value in fp64,
    products and sums in the library's order, rounded once to dtype (np.float64: not rounded).  points [..., 3], depth [...],
    ext [..., 3, 4] world-to-camera; returns the ones given."""
    A, t = np.asarray(sim3, np.float64)[:3, :3], np.asarray(sim3, np.float64)[:3, 3]
    c = np.sqrt(_dot3(A[0, 0], A[1, 0], A[2, 0], A[0, 0], A[1, 0], A[2, 0]))
    out = {}
    if points is not None:
        q = np.asarray(points).astype(np.float64)
        out["points"] = np.stack([_dot3(A[r, 0], A[r, 1], A[r, 2], q[..., 0], q[..., 1], q[..., 2]) + t[r]
                                  for r in range(3)], -1).astype(dtype)
    if depth is not None:
        out["depth"] = (c * np.asarray(depth).astype(np.float64)).astype(dtype)
    if ext is not None:
        e = np.asarray(ext).astype(np.float64)
        R = A / c
        Rp = np.stack([np.stack([_dot3(e[..., r, 0], e[..., r, 1], e[..., r, 2], R[j, 0], R[j, 1], R[j, 2]) for j in range(3)], -1)
                       for r in range(3)], -2)
        tp = np.stack([c * e[..., r, 3] - _dot3(Rp[..., r, 0], Rp[..., r, 1], Rp[..., r, 2], t[0], t[1], t[2]) for r in range(3)], -1)
        out["ext"] = np.concatenate([Rp, tp[..., None]], -1).astype(dtype)
    return out


def unproject(depth: np.ndarray, K: np.ndarray, ext: np.ndarray) -> np.ndarray:
    """fp64 world points [S, H, W, 3] of depth [S, H, W] through pinhole K [S, 3, 3] and world-to-camera ext [S, 3, 4]."""
    d = np.asarray(depth, np.float64)
    S, H, W = d.shape
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    out = []
    for s in range(S):
        k, e = np.asarray(K[s], np.float64), np.asarray(ext[s], np.float64)
        cam = np.stack([(u - k[0, 2]) * d[s] / k[0, 0], (v - k[1, 2]) * d[s] / k[1, 1], d[s]], -1)
        out.append((cam - e[:, 3]) @ e[:, :3])          # R^T (x - t)
    return np.stack(out)


POINT_KEYS = ("world_points_from_depth", "world_points")
COPY_KEYS = ("intrinsic", "depth_conf", "world_points_conf")


def merge(raw: Callable[[int, int], Dict[str, np.ndarray]], S: int, chunk: int, overlap: int, source: str = "depth",
          conf_percent: float = 50.0, threshold: Optional[Callable[[np.ndarray], float]] = None) -> Dict[str, object]:
    """OmniVGGT.reconstruct on given per-chunk outputs: raw(start, end) -> numpy dict of that chunk's views with extrinsic
    [n, 3, 4], intrinsic, depth [n, H, W, 1], depth_conf, world_points_from_depth [n, H, W, 3] and, when the point head is
    set, world_points and world_points_conf.  threshold(conf) -> fp32 percentile threshold (default np.percentile)."""
    chunks = schedule(S, chunk, overlap)
    merged: Dict[str, np.ndarray] = {}
    sims, pairs, rmse = [], [], []
    pkey, ckey = ("world_points_from_depth", "depth_conf") if source == "depth" else ("world_points", "world_points_conf")
    thr = (lambda c: None) if threshold is None else threshold
    for k, ((a, b), (n0, n1)) in enumerate(zip(chunks, new_views(chunks))):
        r = raw(a, b)
        if k == 0:
            merged = {key: np.concatenate([v, np.zeros((S - len(v),) + v.shape[1:], v.dtype)]) for key, v in r.items()}
            sims.append(np.eye(4))
            pairs.append(0.0)
            rmse.append(0.0)
            continue
        ov = slice(0, n0 - a)                                        # the chunk's views already merged
        keep = (keep_mask(r[ckey][ov], conf_percent, threshold=thr(r[ckey][ov]))
                & keep_mask(merged[ckey][a:n0], conf_percent, threshold=thr(merged[ckey][a:n0])))
        sim3, stats = umeyama(r[pkey][ov].reshape(-1, 3), merged[pkey][a:n0].reshape(-1, 3), keep.reshape(-1))
        if stats[1] != STATUS_OK:
            raise ValueError(f"chunk {k} (views {a}..{b - 1}): degenerate overlap, status {int(stats[1])}")
        new = slice(n0 - a, b - a)
        for key in POINT_KEYS:
            if key in r:
                merged[key][n0:n1] = apply(sim3, points=r[key][new])["points"]
        merged["depth"][n0:n1] = apply(sim3, depth=r["depth"][new])["depth"]
        merged["extrinsic"][n0:n1] = apply(sim3, ext=r["extrinsic"][new])["ext"]
        for key in COPY_KEYS:
            if key in r:
                merged[key][n0:n1] = r[key][new]
        sims.append(sim3)
        pairs.append(stats[0])
        rmse.append(stats[2])
    merged.update(chunks=chunks, sim3=np.stack(sims), align_pairs=np.array(pairs), align_rmse=np.array(rmse))
    return merged
