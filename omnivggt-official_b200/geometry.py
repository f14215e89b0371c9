"""Dense correspondence between point maps on the device (libovg ovg_match_*): the reference's
omnivggt/utils/geometry.py:435-451 find_reciprocal_matches."""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def _check_shape(P, name: str) -> None:
    shape = tuple(P.shape) if hasattr(P, "shape") else np.shape(P)
    if len(shape) != 2 or shape[1] != 3:
        raise ValueError(f"{name} must have shape [n, 3], got {shape}")


def find_reciprocal_matches(P1, P2):
    """Drop-in for geometry.py:435-451: the nearest neighbour of every point of P2 among P1 and of every point of P1 among P2,
    and the mutual pairs.  P1 [n, 3], P2 [m, 3]: CUDA tensors, or arrays (moved to the current CUDA device); used as fp32.

    Returns (reciprocal_in_P2 bool [m], nn2_in_P1 int64 [m], count int) with the tensors on the device.  Distances are
    fp64 and computed as cKDTree computes them; among neighbours at the same distance the lowest index wins (cKDTree's choice
    among exact ties is unspecified).  Non-finite points raise ValueError, as cKDTree does.  Unlike the reference, an empty
    P1 or P2 gives zero matches (the reference raises IndexError)."""
    _check_shape(P1, "P1")
    _check_shape(P2, "P2")
    dev = next((p.device for p in (P1, P2) if torch.is_tensor(p) and p.is_cuda), None)
    dev = dev if dev is not None else torch.device("cuda", torch.cuda.current_device())
    a, b = (torch.as_tensor(np.asarray(p) if not torch.is_tensor(p) else p).to(dev, torch.float32) for p in (P1, P2))
    n, m = a.shape[0], b.shape[0]
    if n == 0 or m == 0:
        return torch.zeros(m, device=dev, dtype=torch.bool), torch.zeros(m, device=dev, dtype=torch.int64), 0
    cap = max(n, m)
    pts = torch.zeros(2, cap, 3, device=dev, dtype=torch.float32)
    pts[0, :n], pts[1, :m] = a, b
    keep = torch.zeros(2, cap, device=dev, dtype=torch.uint8)
    keep[0, :n], keep[1, :m] = 1, 1
    mt = ops.Matcher(pts, keep, torch.tensor([[0, 1]], dtype=torch.int32).to(dev))
    reciprocal, nn = mt.pair(0, m)
    counts, nonfinite = mt.counts()
    if nonfinite:
        raise ValueError("data must be finite, check for nan or inf values")
    return reciprocal, nn, counts[0]


def check_pairs(pairs, S: int):
    """[(i, j)] as an int32 array [P, 2]; every i < j of S views when pairs is None."""
    if pairs is None:
        pairs = [(i, j) for i in range(S) for j in range(i + 1, S)]
    out = []
    for p in pairs:
        if len(p) != 2:
            raise ValueError(f"a pair is (i, j), got {p!r}")
        i, j = int(p[0]), int(p[1])
        if not (0 <= i < S and 0 <= j < S):
            raise IndexError(f"pair ({i}, {j}) out of range for {S} views")
        if i == j:
            raise ValueError(f"pair ({i}, {j}) matches a view with itself")
        out.append((i, j))
    return np.array(out, dtype=np.int32).reshape(-1, 2)
