"""Geometry of point maps on the device: dense correspondence (libovg ovg_match_*, the reference's
omnivggt/utils/geometry.py:435-451 find_reciprocal_matches), triangle meshes (libovg ovg_mesh_*, the reference's
omnivggt/viz.py:40-89 pts3d_to_trimesh and cat_meshes), model-free sky segmentation (libovg ovg_segment_sky, the
reference's omnivggt/viz.py:357-393 segment_sky), farthest point sampling (libovg ovg_farthest_point_sample, the
reference's omnivggt/utils/po_utils/misc.py:114-148 farthest_point_sample), the ranking of views by camera distance
(libovg ovg_compute_ranking, the reference's omnivggt/datasets/utils/image_ranking.py:118-140 compute_ranking) and the
similarity alignment of corresponding points (libovg ovg_sim3_estimate, Umeyama's method as the reference's
omnivggt/utils/vo_eval.py:190-233 reaches it through evo)."""
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


def segment_sky(image):
    """Drop-in for viz.py:357-393: the sky of one image.  image [H, W, 3] of dtype uint8, float32 or float64: a CUDA or CPU
    tensor, or an array (moved to the current CUDA device).  Floating images become uint8(255 * clip(x, 0, 1)) in their own
    dtype, truncated (float64 by torch on the device, float32 inside the kernel); channel 0 is read as B, as the reference's
    cv2.cvtColor(..., COLOR_BGR2HSV) does.  Returns bool [H, W] on the device, True = sky."""
    shape = tuple(image.shape) if hasattr(image, "shape") else np.shape(image)
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"image must have shape [H, W, 3], got {shape}")
    dtype = image.dtype if torch.is_tensor(image) else np.asarray(image).dtype
    ok = (dtype in (torch.uint8, torch.float32, torch.float64) if torch.is_tensor(image)
          else dtype in (np.uint8, np.float32, np.float64))
    if not ok:
        raise ValueError(f"image dtype must be uint8, float32 or float64, got {dtype}")
    H, W = shape[:2]
    if H == 0 or W == 0:
        return torch.zeros(H, W, device=_device_of(image), dtype=torch.bool)
    img = _to(image, _device_of(image))
    if img.dtype == torch.float64:
        img = (255 * img.clamp(0, 1)).to(torch.uint8)
    img = img.contiguous()
    sky, _ = ops.segment_sky(img, 1, H, W, H * W * 3, 3, 1)
    return sky.view(H, W).bool()


def farthest_point_sample(xyz, npoint: int, include_ends: bool = False, deterministic: bool = False):
    """Drop-in for po_utils/misc.py:114-148: npoint indices of each batch of xyz [B, N, 3] (a CUDA or CPU tensor, or an array,
    moved to the current CUDA device and used as fp32), each the point farthest from the ones before it.  Returns int64
    [B, npoint] on the device, in selection order.

    The first index is 0 when deterministic, else torch.randint(0, N, (B,)) from torch's default CPU generator, drawn as the
    reference draws it: the same torch.manual_seed gives the same indices.  With include_ends the first two are 0 and N-1.
    Distances are fp32 ((dx*dx + dy*dy) + dz*dz) without contraction; a NaN distance never replaces a running one; ties go to
    the lowest index.  Limits, each a ValueError before any device work: C != 3; N == 0; npoint < 1; npoint > N (where the
    reference adds torch.randn_like noise at every step, which cannot be reproduced)."""
    shape = tuple(xyz.shape) if hasattr(xyz, "shape") else np.shape(xyz)
    if len(shape) != 3 or shape[2] != 3:
        raise ValueError(f"xyz must have shape [B, N, 3], got {shape}")
    B, N = shape[0], shape[1]
    if N == 0:
        raise ValueError("xyz has no points")
    if int(npoint) < 1 or int(npoint) > N:
        raise ValueError(f"npoint must be in [1, N = {N}], got {npoint}")
    start = torch.randint(0, 1 if deterministic else N, (B,), dtype=torch.long)   # misc.py:127-130, same generator draw
    dev = _device_of(xyz)
    if B == 0:
        return torch.zeros(0, int(npoint), device=dev, dtype=torch.int64)
    pts = _to(xyz, dev).float().contiguous()
    return ops.farthest_point_sample(pts, int(npoint), start.to(dev), include_ends)


RANKING_CHUNKED_ABOVE = 6000     # image_ranking.py:129: the batched path switches to its fp32 chunked formula above this


def compute_ranking(extrinsics, lambda_t: float = 1.0, normalize: bool = True, batched: bool = True, k=None):
    """Drop-in for image_ranking.py:118-140: the camera-distance matrix of N views and, per view, every view from nearest to
    farthest.  extrinsics [N, >=3, >=4] of float32 or float64: a CUDA or CPU tensor, or an array (moved to the current CUDA
    device); R = E[:, :3, :3], t = E[:, :3, 3], whatever convention they use.  Returns (ranking int64 [N, k], dists [N, N])
    on the device.

    d(i, j) = degrees(arccos(clip((trace(R_i^T R_j) - 1) / 2, -1, 1))) / 180 + lambda_t |t_i - t_j|, after t / mean |t| when
    normalize.  dists has the reference's dtype: the input's when batched and N <= 6000, float32 when batched and N > 6000
    (computed from float32 operands, as the chunked path is), float64 when not batched.  Each entry is evaluated in fp64
    and rounded once; where the reference computes in float32 (a float32 input, or the chunked path), lambda_t is rounded
    to float32 as numpy does.  ranking is the stable argsort of dists: ties in index order, NaN last (the reference's
    quicksort leaves the order of ties unspecified).  k=None returns every column; k=m returns the first m columns of the
    same ranking, and dists in full.  Limits, each a ValueError before any device work: not 3-D, fewer than 3 rows or 4
    columns, a dtype other than float32 / float64, k outside [1, N]."""
    shape = tuple(extrinsics.shape) if hasattr(extrinsics, "shape") else np.shape(extrinsics)
    if len(shape) != 3 or shape[1] < 3 or shape[2] < 4:
        raise ValueError(f"extrinsics must have shape [N, >=3, >=4], got {shape}")
    dtype = extrinsics.dtype if torch.is_tensor(extrinsics) else np.asarray(extrinsics).dtype
    if dtype not in (torch.float32, torch.float64, np.float32, np.float64):
        raise ValueError(f"extrinsics dtype must be float32 or float64, got {dtype}")
    in_f64 = dtype in (torch.float64, np.float64)
    N = shape[0]
    if k is None:
        k = N
    elif isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= N:
        raise ValueError(f"k must be an integer in [1, N = {N}], got {k!r}")
    if not batched:
        out = torch.float64
    elif N > RANKING_CHUNKED_ABOVE:
        out = torch.float32
    else:
        out = torch.float64 if in_f64 else torch.float32
    lam = float(lambda_t) if in_f64 and out == torch.float64 else float(np.float32(lambda_t))
    dev = _device_of(extrinsics)
    if N == 0:
        return torch.zeros(0, 0, device=dev, dtype=torch.int64), torch.zeros(0, 0, device=dev, dtype=out)
    return ops.compute_ranking(_to(extrinsics, dev), lam, normalize, out, int(k))


SIM3_STATUS = {1: "fewer than 3 kept pairs", 2: "the source points all coincide (sigma^2 == 0)",
               3: "the points are collinear or coincide (second singular value <= 1e-12 x the first)"}


def align_sim3(src, dst, keep=None):
    """The similarity transform that best maps src onto dst: fp64 [4, 4] [[c R, t], [0, 1]] on the device, minimising
    sum |dst - (c R src + t)|^2 over the kept pairs (Umeyama 1991, eqs. 40-42; what evo's umeyama_alignment computes with
    correct_scale, and what the reference's vo_eval reaches through align=True, correct_scale=True).

    src, dst [N, 3]: CUDA tensors, or arrays (moved to the current CUDA device), used as fp32.  keep [N] (bool or integer,
    non-zero = kept) or None.  Pairs with a non-finite coordinate are dropped.  Aligns predicted point maps to ground truth,
    or a predicted trajectory of camera centres to a reference one (the ATE alignment).  Raises ValueError when fewer than 3
    pairs are kept or the kept points are coincident or collinear; reading that status is the call's one host read."""
    _check_shape(src, "src")
    _check_shape(dst, "dst")
    n = (src.shape if hasattr(src, "shape") else np.shape(src))[0]
    if (dst.shape if hasattr(dst, "shape") else np.shape(dst))[0] != n:
        raise ValueError("src and dst must have the same number of points")
    if keep is not None and tuple(keep.shape if hasattr(keep, "shape") else np.shape(keep)) != (n,):
        raise ValueError(f"keep must have shape [{n}]")
    dev = _device_of(src, dst, keep)
    s, d = (_to(p, dev).to(torch.float32).contiguous() for p in (src, dst))
    k = None if keep is None else (_to(keep, dev) != 0).to(torch.uint8).contiguous()
    sim3, stats = ops.sim3_estimate(s, d, k)
    status = int(ops.host_read(stats[1]))
    if status:
        raise ValueError(f"align_sim3: degenerate input: {SIM3_STATUS[status]}")
    return sim3


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
