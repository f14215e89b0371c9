"""Geometry of point maps on the device: dense correspondence (libovg ovg_match_*, the reference's
omnivggt/utils/geometry.py:435-451 find_reciprocal_matches) and triangle meshes (libovg ovg_mesh_*, the reference's
omnivggt/viz.py:40-89 pts3d_to_trimesh and cat_meshes)."""
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


def _device_of(*xs):
    dev = next((x.device for x in xs if torch.is_tensor(x) and x.is_cuda), None)
    return dev if dev is not None else torch.device("cuda", torch.cuda.current_device())


def _to(x, dev):
    return (x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))).to(dev)


def pts3d_to_trimesh(img, pts3d, valid=None):
    """Drop-in for viz.py:40-77: the triangle mesh of one point map.  img [H, W, 3] (uint8, float32 or any dtype of 1, 2, 4
    or 8 bytes), pts3d [H, W, 3], valid [H, W] or None: CUDA tensors, or arrays (moved to the current CUDA device).

    Returns ``{"vertices", "face_colors", "faces"}`` on the device: vertices = pts3d as [H*W, 3] in its dtype; faces int64
    [n, 3], per pixel quad (tl, tr, bl), its reverse, (tr, bl, br), its reverse, each class in row-major order, keeping a face
    when its three pixels are valid (every face when valid is None); face_colors [n, 3] gathered from img without arithmetic
    (tl's colour for the first two classes, br's for the last two), so they keep img's dtype."""
    shape = tuple(img.shape)
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"img must have shape [H, W, 3], got {shape}")
    if tuple(pts3d.shape) != shape:
        raise ValueError(f"pts3d must have the shape of img {shape}, got {tuple(pts3d.shape)}")
    if valid is not None and tuple(valid.shape) != shape[:2]:
        raise ValueError(f"valid must have shape {shape[:2]}, got {tuple(valid.shape)}")
    H, W = shape[:2]
    dev = _device_of(img, pts3d, valid)
    colors = _to(img, dev).contiguous()
    if colors.element_size() not in (1, 2, 4, 8):
        raise ValueError(f"img dtype {colors.dtype} is not 1, 2, 4 or 8 bytes wide")
    pts = _to(pts3d, dev)
    keep = (torch.ones(H * W, device=dev, dtype=torch.uint8) if valid is None
            else (_to(valid, dev) != 0).to(torch.uint8).reshape(-1).contiguous())
    mesher = ops.Mesher(keep, None, 1, H, W)
    n = int(ops.host_read(mesher.totals)[0])
    faces, face_colors = mesher.faces(n, colors.view(H * W, 3))
    return {"vertices": pts.reshape(-1, 3), "face_colors": face_colors, "faces": faces}


def cat_meshes(meshes):
    """Drop-in for viz.py:80-89: vertices and face colours concatenated, each mesh's faces offset by the vertices of the
    meshes before it; tensors on the device.  Unlike the reference, the inputs' faces are not modified in place."""
    meshes = list(meshes)
    if not meshes:
        raise ValueError("need at least one mesh")
    dev = _device_of(*(m["faces"] for m in meshes))
    n = 0
    faces = []
    for m in meshes:
        faces.append(_to(m["faces"], dev) + n)
        n += len(m["vertices"])
    return {"vertices": torch.cat([_to(m["vertices"], dev) for m in meshes]),
            "face_colors": torch.cat([_to(m["face_colors"], dev) for m in meshes]),
            "faces": torch.cat(faces)}
