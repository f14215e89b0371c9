"""Farthest point sampling restated (po_utils/misc.py:114-148, farthest_point_sample): numpy on the host, and the same loop
in torch for CUDA tensors, each vectorised over the batches per step.  Neither reads the reference.

Per batch: distance starts at fp32 1e10; step i records inds[:, i] = farthest (with include_ends, 0 at i = 0 and N-1 at
i = 1), then d = ((dx*dx + dy*dy) + dz*dz) in fp32 with every operation rounded, distance = d where d < distance (a NaN d
never updates), and farthest = the first index of the largest distance."""
from __future__ import annotations

import numpy as np


def farthest_point_sample(xyz, npoint: int, include_ends: bool = False, start=None) -> np.ndarray:
    """xyz [B, N, 3] (cast to fp32), start int64 [B] (None: zeros) -> int64 [B, npoint]."""
    p = np.asarray(xyz).astype(np.float32)
    B, N, _ = p.shape
    far = np.zeros(B, np.int64) if start is None else np.array(start, np.int64).reshape(B)
    dist = np.full((B, N), np.float32(1e10), np.float32)
    out = np.zeros((B, npoint), np.int64)
    rows = np.arange(B)
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(npoint):
            if include_ends and i < 2:
                far[:] = 0 if i == 0 else N - 1
            out[:, i] = far
            q = p - p[rows, far][:, None, :]
            q = q * q
            d = (q[..., 0] + q[..., 1]) + q[..., 2]
            dist = np.where(d < dist, d, dist)
            far = np.argmax(dist, axis=1)
    return out


def farthest_point_sample_torch(xyz, npoint: int, include_ends: bool = False, start=None):
    """The same loop on torch tensors (CUDA or CPU): xyz [B, N, 3], start int64 [B] on xyz's device (None: zeros).  One
    elementwise kernel per operation, so nothing is contracted; torch.argmax returns the first maximal index."""
    import torch
    p = xyz.float()
    B, N, _ = p.shape
    far = torch.zeros(B, dtype=torch.long, device=p.device) if start is None else start.to(p.device, torch.long).clone()
    dist = torch.full((B, N), 1e10, dtype=torch.float32, device=p.device)
    out = torch.zeros(B, npoint, dtype=torch.long, device=p.device)
    rows = torch.arange(B, device=p.device)
    for i in range(npoint):
        if include_ends and i < 2:
            far.fill_(0 if i == 0 else N - 1)
        out[:, i] = far
        q = p - p[rows, far][:, None, :]
        q = q * q
        d = (q[..., 0] + q[..., 1]) + q[..., 2]
        dist = torch.where(d < dist, d, dist)
        far = torch.argmax(dist, dim=1)
    return out
