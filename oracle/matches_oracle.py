"""numpy restatement of reciprocal nearest-neighbour matching (reference omnivggt/utils/geometry.py:435-451
find_reciprocal_matches, :15-37 xy_grid) under the contract libovg's ovg_match_* implement:

  - points are fp32; squared distances are fp64, d2 = ((dx*dx) + (dy*dy)) + dz*dz with dx = double(q.x) - double(p.x) (what
    cKDTree computes for 3-D data);
  - the nearest neighbour is the lowest index among the points at the smallest d2 (cKDTree's choice among exact ties is
    unspecified);
  - reciprocal_in_P2[j] = nn1_in_P2[nn2_in_P1[j]] == j;
  - an empty set gives no matches.

nn_brute is the definition (np.argmin takes the lowest index), for up to about 20 k points; nn_kdtree gets the same answer
for large sets from cKDTree plus an explicit resolution of ties."""
from __future__ import annotations

import numpy as np


def d2_of(Q: np.ndarray, T: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """fp64 d2 between Q[k] and T[idx[k]], in the contract's order of operations."""
    q = Q.astype(np.float64)
    t = T.astype(np.float64)[idx]
    d = q - t
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def nn_brute(Q: np.ndarray, T: np.ndarray, chunk: int = 256):
    """(idx int64 [n], d2 fp64 [n]): nearest neighbour of every point of Q among T, lowest index among ties."""
    Q = np.asarray(Q, np.float32)
    T = np.asarray(T, np.float32)
    t = T.astype(np.float64)
    idx = np.empty(len(Q), np.int64)
    best = np.empty(len(Q), np.float64)
    for s in range(0, len(Q), chunk):
        q = Q[s:s + chunk].astype(np.float64)
        dx = q[:, None, 0] - t[None, :, 0]
        dy = q[:, None, 1] - t[None, :, 1]
        dz = q[:, None, 2] - t[None, :, 2]
        d2 = (dx * dx + dy * dy) + dz * dz
        i = np.argmin(d2, axis=1)
        idx[s:s + chunk] = i
        best[s:s + chunk] = d2[np.arange(len(q)), i]
    return idx, best


def nn_kdtree(Q: np.ndarray, T: np.ndarray):
    """nn_brute for large sets: cKDTree's two nearest neighbours; where they are at the same d2, every point within that
    distance is examined and the lowest index at the smallest d2 is taken."""
    from scipy.spatial import cKDTree
    Q = np.asarray(Q, np.float32)
    T = np.asarray(T, np.float32)
    tree = cKDTree(T)
    k = min(2, len(T))
    dist, idx = tree.query(Q, k=k, workers=-1)
    idx = idx.reshape(len(Q), k)
    d2 = np.stack([d2_of(Q, T, idx[:, c]) for c in range(k)], 1)
    out, best = idx[:, 0].copy(), d2[:, 0].copy()
    if k == 2:
        for q in np.flatnonzero(d2[:, 1] <= d2[:, 0]):
            cand = np.array(tree.query_ball_point(Q[q], np.nextafter(np.sqrt(best[q]), np.inf) * (1 + 1e-12)), np.int64)
            cd = d2_of(np.repeat(Q[q:q + 1], len(cand), 0), T, cand)
            m = cd.min()
            out[q], best[q] = cand[cd == m].min(), m
    return out.astype(np.int64), best


def find_reciprocal_matches(P1, P2, nn=nn_brute):
    """(reciprocal_in_P2 bool [m], nn2_in_P1 int64 [m], count int), geometry.py:442-451 under the contract."""
    P1 = np.asarray(P1, np.float32).reshape(-1, 3)
    P2 = np.asarray(P2, np.float32).reshape(-1, 3)
    if len(P1) == 0 or len(P2) == 0:
        return np.zeros(len(P2), bool), np.zeros(len(P2), np.int64), 0
    nn1_in_P2, _ = nn(P1, P2)
    nn2_in_P1, _ = nn(P2, P1)
    reciprocal_in_P2 = nn1_in_P2[nn2_in_P1] == np.arange(len(P2))
    return reciprocal_in_P2, nn2_in_P1, int(reciprocal_in_P2.sum())


def has_ties(Q: np.ndarray, T: np.ndarray) -> bool:
    """Whether some point of Q has two points of T at its smallest d2."""
    from scipy.spatial import cKDTree
    if len(T) < 2 or len(Q) == 0:
        return False
    _, idx = cKDTree(np.asarray(T, np.float32)).query(np.asarray(Q, np.float32), k=2, workers=-1)
    return bool((d2_of(Q, T, idx[:, 1]) <= d2_of(Q, T, idx[:, 0])).any())


def xy_grid(W: int, H: int) -> np.ndarray:
    """geometry.py:15-37 (numpy): int [H, W, 2] with grid[y, x] = (x, y)."""
    return np.stack(np.meshgrid(np.arange(W), np.arange(H), indexing="xy"), -1)


def scene_matches(points: np.ndarray, keep: np.ndarray, pairs, nn=nn_brute):
    """The DUSt3R recipe per pair (i, j): P1, P2 = kept points of views i, j (row-major); xy_j = grid[kept_j][reciprocal_in_P2],
    xy_i = grid[kept_i][nn2_in_P1][reciprocal_in_P2].  points [S, H, W, 3], keep bool [S, H, W]."""
    S, H, W, _ = points.shape
    grid = xy_grid(W, H).reshape(-1, 2).astype(np.int64)
    pts = points.reshape(S, H * W, 3)
    kp = keep.reshape(S, H * W)
    out = []
    for i, j in pairs:
        rec, nn2, n = find_reciprocal_matches(pts[i][kp[i]], pts[j][kp[j]], nn)
        out.append({"xy_i": grid[kp[i]][nn2][rec], "xy_j": grid[kp[j]][rec], "count": n})
    return out
