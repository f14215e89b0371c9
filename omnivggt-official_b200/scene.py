"""A predictions dict on the device: its cameras and world points (``postprocess``), and the sky, point cloud, mesh,
matches and tracks of one scene.  They read no weight; ``OmniVGGT`` exposes each under the same name.  Each checks its
arguments before any library call (``_check_views``), then takes the scene's views from ``_kept_views``."""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

from . import geometry, ops


def _of_scene(t: torch.Tensor, trailing: int, scene: int) -> torch.Tensor:
    """[B, S, ...] or [S, ...] -> [S, ...] of the scene, for a key with ``trailing`` dimensions after the view."""
    return t[scene] if t.dim() == trailing + 2 else t


def decode_cameras(pose_enc: torch.Tensor, depth: Optional[torch.Tensor], H: int, W: int):
    """(extrinsic fp32 [..., 3, 4], intrinsic fp32 [..., 3, 3], world points fp32 [..., H, W, 3]): the cameras of pose_enc
    [..., 9] (ovg_pose_decode, inference.py:360-365 -> utils/pose_enc.py:65-130) and depth [..., H, W(, 1)] unprojected
    through them (ovg_unproject_depth, visual_util.py:42-73 -> utils/geometry.py:151-264); no points when depth is None."""
    ext, intr, c2w = ops.pose_decode(pose_enc.float(), H, W)
    if depth is None:
        return ext, intr, None
    world = ops.unproject_depth(depth.float().reshape(-1, H, W), intr.view(-1, 3, 3), c2w.view(-1, 3, 4), H, W)
    return ext, intr, world.view(*ext.shape[:-2], H, W, 3)


@torch.no_grad()
def postprocess(predictions: Dict[str, object], conf_percent: float = 50.0, use_point_map: bool = False
                ) -> Dict[str, object]:
    """What reference inference.py does on the host right after the forward, on the device (libovg kernels):
    ``extrinsic`` / ``intrinsic`` from ``pose_enc`` (inference.py:360-365 -> utils/pose_enc.py:65-130),
    ``world_points_from_depth`` by unprojecting the predicted depth with the predicted cameras (visual_util.py:42-73 ->
    utils/geometry.py:151-264), and the confidence filter of the viewer (inference.py:132-133): ``conf_mask`` =
    conf >= percentile(conf, conf_percent) & conf > 0.1 with ``conf_threshold`` / ``conf_kept``, over
    ``world_points_conf`` if ``use_point_map`` else ``depth_conf`` (inference.py:95-100).  Adds the keys in place."""
    H, W = predictions["images"].shape[-2:]
    ext, intr, world = decode_cameras(predictions["pose_enc"], predictions["depth"], H, W)
    predictions["extrinsic"], predictions["intrinsic"], predictions["world_points_from_depth"] = ext, intr, world
    conf = predictions["world_points_conf" if use_point_map else "depth_conf"].float()
    mask, thr, cnt = ops.conf_percentile_mask(conf, conf_percent, 0.1)
    predictions["conf_mask"], predictions["conf_threshold"], predictions["conf_kept"] = mask.bool(), thr, cnt
    return predictions


def _check_views(predictions: Dict[str, object], source: str, conf_percent: float, conf_floor: float,
                 frame: Optional[int], scene: int, mask_sky) -> int:
    """The argument checks of point_cloud, mesh, matches and tracks, before any library call; returns the view count."""
    if source not in ("depth", "pointmap"):
        raise ValueError(f"source must be 'depth' or 'pointmap', got {source!r}")
    if not 0.0 <= conf_percent <= 100.0:
        raise ValueError("conf_percent must be in [0, 100]")
    if conf_floor < 0.0:
        raise ValueError("conf_floor must be >= 0")        # the reference's floors are 1e-5 and 0.1
    _check_mask_sky(mask_sky, predictions, scene)
    S = _of_scene(predictions["images"], 3, scene).shape[0]
    if frame is not None and not 0 <= frame < S:
        raise IndexError(f"frame {frame} out of range for {S} views")
    return S


def _check_mask_sky(mask_sky, predictions: Dict[str, object], scene: int) -> None:
    """mask_sky is a bool, or a bool tensor [S, H, W] / [B, S, H, W] (True = sky) on the images' device."""
    if isinstance(mask_sky, (bool, np.bool_)):
        return
    if not torch.is_tensor(mask_sky) or mask_sky.dtype != torch.bool:
        raise ValueError(f"mask_sky must be a bool or a bool tensor, got {getattr(mask_sky, 'dtype', type(mask_sky))}")
    images = predictions["images"]
    S, _, H, W = _of_scene(images, 3, scene).shape
    full = [images.shape[0], S, H, W] if images.dim() == 5 else None
    if list(mask_sky.shape) not in ([S, H, W], full):
        raise ValueError(f"mask_sky must have shape [S, H, W] = {[S, H, W]}" + (f" or [B, S, H, W] = {full}" if full else "")
                         + f", got {list(mask_sky.shape)}")
    if mask_sky.device != images.device:
        raise ValueError(f"mask_sky is on {mask_sky.device}, the images on {images.device}")


def _kept_views(predictions: Dict[str, object], source: str, conf_percent: float, conf_floor: float,
                frame: Optional[int], scene: int, mask_sky, cameras: Optional[str] = None):
    """The views point_cloud, mesh, matches and tracks work on, after _check_views: the scene's source, its confidence
    times non-sky over all views (visual_util.py:186-188; no launch without mask_sky), then the frame, then
    conf >= percentile(conf, conf_percent) and conf > conf_floor.
    ``source="depth"``: ``world_points_from_depth`` with ``depth_conf``; ``"pointmap"``: ``world_points`` with
    ``world_points_conf``.  Returns (images fp32 [F,3,H,W], cameras, points fp32 [F,H,W,3], mask uint8 [F,H,W],
    threshold 0-d, first view f0), the images, points and mask contiguous; the cameras fp32 [S,3,4] / [S,3,3] contiguous.

    Points and cameras by the keys the predictions hold.  ``pose_enc`` is decoded once at most, and only when a row below
    needs it:
      points                 ``source="depth"`` without ``world_points_from_depth``: the depth unprojected through the
                             decoded intrinsic and cam2world, never through the predictions' own cameras.
      cameras=None           () (matches).
      cameras="points"       (extrinsic,) of the camera the points are in (align's E0 in point_cloud and mesh): the
                             decoded one when the depth is unprojected here, else the predictions' own, else the decoded one.
      cameras="predictions"  (extrinsic, intrinsic) (tracks): the predictions' own, each on its own; the decoded one for
                             whichever is missing."""
    images = _of_scene(predictions["images"], 3, scene).float()
    _, _, H, W = images.shape
    pkey, ckey = ("world_points", "world_points_conf") if source == "pointmap" else ("world_points_from_depth", "depth_conf")
    unproject = source == "depth" and pkey not in predictions
    own = {k: _of_scene(predictions[k], 2, scene) for k in ("extrinsic", "intrinsic") if k in predictions}
    if cameras == "points" and unproject:
        own = {}                                            # E0 is then the camera the depth is unprojected through
    want = {None: (), "points": ("extrinsic",), "predictions": ("extrinsic", "intrinsic")}[cameras]
    decoded = {}
    if unproject or any(k not in own for k in want):
        depth = _of_scene(predictions["depth"], 3, scene) if unproject else None
        decoded["extrinsic"], decoded["intrinsic"], points = decode_cameras(_of_scene(predictions["pose_enc"], 1, scene),
                                                                            depth, H, W)
    if not unproject:
        points = _of_scene(predictions[pkey], 3, scene)
    cams = tuple(own[k].float().contiguous() if k in own else decoded[k] for k in want)
    conf = _of_scene(predictions[ckey], 2, scene)
    if torch.is_tensor(mask_sky):
        conf = ops.sky_mask_conf(conf.float().contiguous(), _of_scene(mask_sky, 2, scene).contiguous().view(torch.uint8))
    elif mask_sky:
        _, conf = _segment_views(images, conf.float().contiguous())
    f0 = 0 if frame is None else frame
    if frame is not None:
        images, points, conf = images[frame:frame + 1], points[frame:frame + 1], conf[frame:frame + 1]
    mask, thr, _ = ops.conf_percentile_mask(conf.float().contiguous(), conf_percent, conf_floor)
    if conf_percent == 0.0:
        thr = torch.zeros((), device=images.device, dtype=torch.float32)   # same mask: conf > conf_floor >= 0 implies conf >= 0
    return images.contiguous(), cams, points.float().contiguous(), mask, thr, f0


def _segment_views(images: torch.Tensor, conf: Optional[torch.Tensor] = None):
    """ops.segment_sky over the views of images fp32 [S,3,H,W], read in place when each channel plane is contiguous."""
    S, _, H, W = images.shape
    if images.stride(3) != 1 or images.stride(2) != W:
        images = images.contiguous()
    return ops.segment_sky(images, S, H, W, images.stride(0), 1, images.stride(1), conf)


@torch.no_grad()
def sky_mask(predictions: Dict[str, object], *, scene: int = 0) -> torch.Tensor:
    """The sky of every view of one scene: the reference's model-free segment_sky (viz.py:357-393) on the images the model
    saw, ``predictions["images"]`` fp32 [S,3,H,W] (or [B,S,3,H,W]), all views in one call with no host read.  Returns bool
    [S, H, W] on the device, True = sky; ``point_cloud``, ``mesh`` and ``matches`` take it as ``mask_sky``."""
    sky, _ = _segment_views(_of_scene(predictions["images"], 3, scene).float())
    return sky.bool()


@torch.no_grad()
def matches(predictions: Dict[str, object], pairs=None, *, source: str = "depth", conf_percent: float = 50.0,
            conf_floor: float = 1e-5, scene: int = 0, mask_sky=False) -> List[Dict[str, object]]:
    """Dense cross-view correspondences of one scene by reciprocal nearest neighbours of the predicted points (the
    DUSt3R-family recipe on utils/geometry.py:435-451 find_reciprocal_matches and :15-37 xy_grid), on the device.

    ``source`` and the keep mask are ``point_cloud``'s: conf >= percentile(conf over the scene's S views, conf_percent) and
    conf > conf_floor.  For each pair (i, j) (default: every i < j), P1 and P2 are the kept points of views i and j in
    row-major order, and the result is ``{"xy_i", "xy_j", "count"}`` with ``xy_j = grid_j[kept_j][reciprocal_in_P2]`` and
    ``xy_i = grid_i[kept_i][nn2_in_P1][reciprocal_in_P2]``: int64 [count, 2] (x, y) pixel coordinates on the device.
    Every view's index is built once; all pairs are queried in one pass; the match counts are the one host read.  Kept
    points that are not finite raise ValueError; a view with no kept point has no matches.  ``mask_sky``: as in
    ``point_cloud``."""
    S = _check_views(predictions, source, conf_percent, conf_floor, None, scene, mask_sky)
    pair_arr = geometry.check_pairs(pairs, S)
    if len(pair_arr) == 0:
        return []
    images, _, points, mask, _, _ = _kept_views(predictions, source, conf_percent, conf_floor, None, scene, mask_sky)
    _, _, H, W = images.shape
    mt = ops.Matcher(points.view(S, H * W, 3), mask.view(S, H * W), torch.from_numpy(pair_arr).to(images.device))
    counts, nonfinite = mt.counts()
    if nonfinite:
        raise ValueError("kept points must be finite (cKDTree: data must be finite, check for nan or inf values)")
    xy_i, xy_j = mt.gather(sum(counts), W)
    return [{"xy_i": a, "xy_j": b, "count": c} for a, b, c in zip(xy_i.split(counts), xy_j.split(counts), counts)]


@torch.no_grad()
def tracks(predictions: Dict[str, object], pairs=None, *, source: str = "depth", conf_percent: float = 50.0,
           conf_floor: float = 1e-5, scene: int = 0, mask_sky=False, min_views: int = 2) -> Dict[str, torch.Tensor]:
    """Multi-view tracks of one scene for a COLMAP sparse model (``colmap.write_colmap``), built on the device from the
    reciprocal matches of ``matches``; no counterpart in the reference.

    ``source``, the keep mask, ``mask_sky`` and ``pairs`` are those of ``matches``; (i, j) and (j, i) are one pair and
    duplicates are merged.  Star tracks: views anchor in order a = 0 .. S-1; every kept pixel of view a not yet in a
    track gathers its partners, its reciprocal match in each view j > a of a pair (a, j) that is not in a track either,
    and when 1 + partners >= ``min_views`` (in [1, S]; 1 turns every remaining kept pixel into a one-view point) they
    become one new track.  Tracks are numbered by (anchor view, anchor pixel in row-major order); each has at most one
    observation per view, in ascending view order, and every pixel is in at most one track.  Matches are not chained
    across pairs: reciprocal nearest neighbours of different pairs are not transitive.

    Returns on the device, per track: ``points`` fp64 [n, 3] (the mean of the observations' points, not rounded to
    fp32), ``colors`` uint8 [n, 3] (the anchor pixel's, as ``point_cloud`` computes colours), ``error`` fp64 [n] (mean
    reprojection distance in pixels, COLMAP's pixel-centre convention, +inf when a camera sees the point behind it) and
    ``offsets`` int64 [n + 1]; per observation: ``view`` int32 [m], ``xy`` int64 [m, 2] (x, y) and ``point2d`` int32
    [m] (rank of the pixel in its view's list); per view: ``view_offsets`` int64 [S + 1], ``view_track`` int32 [m] and
    ``view_xy`` int64 [m, 2], each view's pixels in tracks in row-major order; and the ``extrinsic`` / ``intrinsic``
    used, decoded from ``pose_enc`` where the predictions do not hold them.  The counts are the one host read; kept
    points that are not finite raise ValueError."""
    S = _check_views(predictions, source, conf_percent, conf_floor, None, scene, mask_sky)
    if not geometry._is_int(min_views) or not 1 <= min_views <= S:
        raise ValueError(f"min_views must be an integer in [1, {S}], got {min_views!r}")
    pair_arr = geometry.check_pairs(pairs, S)
    pair_arr = np.unique(np.sort(pair_arr, axis=1), axis=0).astype(np.int32).reshape(-1, 2)
    H, W = predictions["images"].shape[-2:]
    if S * H * W >= 2 ** 31:
        raise ValueError(f"tracks need views * H * W < 2^31, got {S} x {H} x {W}")
    if not ("extrinsic" in predictions and "intrinsic" in predictions or "pose_enc" in predictions):
        raise ValueError("tracks need extrinsic and intrinsic, or pose_enc to decode them from")
    images, (ext, intr), points, mask, _, _ = _kept_views(predictions, source, conf_percent, conf_floor, None, scene,
                                                         mask_sky, cameras="predictions")
    # the pairs of anchor a are pair_arr[pair_off[a]:pair_off[a + 1]]; the matcher sizes its workspace by at least one
    # pair, so without pairs it queries view 0 against itself, which no anchor reads
    pair_off = np.searchsorted(pair_arr[:, 0], np.arange(S + 1)).astype(np.int32)
    queried = pair_arr if len(pair_arr) else np.zeros((1, 2), np.int32)
    dev = images.device
    packed = torch.from_numpy(np.concatenate([queried.ravel(), pair_off])).to(dev)
    mt = ops.Matcher(points.view(S, H * W, 3), mask.view(S, H * W), packed[:queried.size].view(-1, 2))
    tr = ops.Tracker(mt, packed[queried.size:], min_views)
    n, m, nonfinite = tr.counts()
    if nonfinite:
        raise ValueError("kept points must be finite (cKDTree: data must be finite, check for nan or inf values)")
    out = tr.gather(images, ext, intr, W, n, m)
    out.update(extrinsic=ext, intrinsic=intr)
    return out


@torch.no_grad()
def point_cloud(predictions: Dict[str, object], *, source: str = "depth", conf_percent: float = 50.0,
                conf_floor: float = 1e-5, frame: Optional[int] = None, mask_black_bg: bool = False,
                mask_white_bg: bool = False, scene: int = 0, mask_sky=False,
                max_points: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """The filtered, coloured point cloud of one scene, built on the device (libovg kernels).

    Replaces the host numpy of the reference's GLB export (visual_util.py:190-236,:320-358 predictions_to_glb) and
    viewer (inference.py:96-151).  ``source="depth"``: ``world_points_from_depth`` (computed here when ``postprocess``
    has not run) with ``depth_conf``, as ``--save_glb`` uses it; ``"pointmap"``: ``world_points`` with
    ``world_points_conf``.  ``frame``: keep only that view, selected before the percentile (visual_util.py:190-194).
    Kept: conf >= percentile(conf, conf_percent) (0 for conf_percent == 0, visual_util.py:206-207) and conf > conf_floor,
    minus black / white background pixels when asked.  ``conf_floor=0.1`` reproduces the viewer's initial mask
    (inference.py:132-133); its frame dropdown is ``cloud["frame"] == i`` on the ``frame=None`` cloud.

    Returns ``points`` fp32 [n,3], ``colors`` uint8 [n,3], ``frame`` int32 [n] (numpy boolean-indexing order),
    ``conf_threshold`` (0-d), ``center`` fp32 [3] (mean of all points of the selected views, inference.py:111),
    ``scale`` (0-d, ||p95 - p5||, 1.0 when nothing is kept) and ``align`` fp64 [4,4] = inv(E0) diag(1,-1,-1,1) R_y(180)
    with E0 the first selected camera (visual_util.py:320-341).  The kept count and E0 are the only device-to-host reads.

    ``mask_sky`` (the reference's --mask_sky, visual_util.py:140-188): False, no sky masking; True, the sky of every view
    by ``sky_mask``; or a bool tensor [S,H,W] / [B,S,H,W], True = sky (a reference mask file m, uint8 255 = non-sky, at
    H x W is ``m == 0``).  The confidence of every view becomes conf * non-sky before the frame selection and the
    percentile, as the reference orders it; no host read is added.

    ``max_points`` (None: every kept point): when more than max_points points are kept, ``points``, ``colors`` and
    ``frame`` are those of the reference's farthest_point_sample (po_utils/misc.py:114-148, deterministic, from the first
    kept point) over the kept points, max_points of them in selection order, so every prefix is a coarser sample of the
    whole cloud.  ``conf_threshold``, ``center``, ``scale`` and ``align`` stay those of all kept points.  A cloud with fewer
    than max_points distinct positions repeats points, as the reference's indices do.  One more launch, no host read."""
    _check_views(predictions, source, conf_percent, conf_floor, frame, scene, mask_sky)
    if max_points is not None and (not geometry._is_int(max_points) or max_points < 1):
        raise ValueError(f"max_points must be None or an integer >= 1, got {max_points!r}")
    images, (ext,), points, mask, thr, f0 = _kept_views(predictions, source, conf_percent, conf_floor, frame, scene,
                                                        mask_sky, cameras="points")
    F, _, H, W = images.shape
    dev = images.device
    ws = ops.point_cloud_workspace(F * H * W, dev)
    cnt = ops.point_cloud_count(mask, images, ws, mask_black_bg, mask_white_bg)
    center = ops.point_cloud_center(points, ws)
    host = ops.host_read(torch.cat([cnt.double().reshape(1), ext[f0].double().reshape(-1)]))   # count < 2^31: exact
    n = int(host[0])
    align = _align(host[1:].view(3, 4)).to(dev)
    if n == 0:
        return {"points": torch.empty(0, 3, device=dev), "colors": torch.empty(0, 3, device=dev, dtype=torch.uint8),
                "frame": torch.empty(0, device=dev, dtype=torch.int32), "conf_threshold": thr, "center": center,
                "scale": torch.ones((), device=dev), "align": align}
    pts, cols, fr, xyz = ops.point_cloud_gather(points, mask, images, ws, n, mask_black_bg, mask_white_bg, f0)
    scale = ops.point_cloud_scale(xyz, n, ws)
    if max_points is not None and n > max_points:
        idx = ops.farthest_point_sample(pts[None], int(max_points), torch.zeros(1, device=dev, dtype=torch.int64))[0]
        pts, cols, fr = pts[idx], cols[idx], fr[idx]
    return {"points": pts, "colors": cols, "frame": fr, "conf_threshold": thr, "center": center, "scale": scale,
            "align": align}


def _align(e0: torch.Tensor) -> torch.Tensor:
    """inv(E0) diag(1,-1,-1,1) R_y(180), fp64 [4,4] on the host, from the host camera E0 [3,4] (visual_util.py:320-341)."""
    e = torch.eye(4, dtype=torch.float64)
    e[:3, :4] = e0
    gl = torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0], dtype=torch.float64))
    rot_y = torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0], dtype=torch.float64))
    return torch.linalg.inv(e) @ gl @ rot_y


@torch.no_grad()
def mesh(predictions: Dict[str, object], *, source: str = "depth", conf_percent: float = 50.0, conf_floor: float = 1e-5,
         frame: Optional[int] = None, mask_black_bg: bool = False, mask_white_bg: bool = False, scene: int = 0,
         layout: str = "reference", mask_sky=False) -> Dict[str, torch.Tensor]:
    """The coloured triangle mesh of one scene's point maps, built on the device (libovg kernels): the DUSt3R-family
    recipe of viz.py:40-89, ``cat_meshes([pts3d_to_trimesh(colors[f], points[f], keep[f]) for f in views])``.

    ``source``, ``conf_percent``, ``conf_floor``, ``frame``, the background masks and ``scene`` select the views and the
    kept pixels exactly as in ``point_cloud``; colours are (images * 255).astype(uint8).  Every pixel quad gives two
    triangles, (tl, tr, bl) and (tr, bl, br); a triangle is kept when its three pixels are.

    ``layout="reference"``: ``vertices`` fp32 [F*H*W, 3] (every point of the selected views), ``face_colors`` uint8 [n, 3]
    and ``faces`` int64 [n, 3], as viz.py returns them: per view the kept (tl, tr, bl) triangles, the same reversed, the kept
    (tr, bl, br) triangles, the same reversed, each in row-major order; colours from tl and br.
    ``layout="glb"``: ``positions`` fp32 [m, 3] and ``colors`` uint8 [m, 3] of the vertices the forward triangles use, in
    index order, each with its own pixel's colour, and ``indices`` int32 [k, 3] of the forward triangles only, for
    ``glb.write_mesh_glb`` (whose material is double-sided in place of the reversed copies).
    Both add ``conf_threshold`` and ``align``, as ``point_cloud`` returns them.  The three totals and the first camera are
    read back together: the one host synchronisation.  ``mask_sky``: as in ``point_cloud``."""
    _check_views(predictions, source, conf_percent, conf_floor, frame, scene, mask_sky)
    if layout not in ("reference", "glb"):
        raise ValueError(f"layout must be 'reference' or 'glb', got {layout!r}")
    images, (ext,), points, mask, thr, f0 = _kept_views(predictions, source, conf_percent, conf_floor, frame, scene,
                                                        mask_sky, cameras="points")
    F, _, H, W = images.shape
    mesher = ops.Mesher(mask.view(-1), images, F, H, W, mask_black_bg, mask_white_bg)
    host = ops.host_read(torch.cat([mesher.totals.double(), ext[f0].double().reshape(-1)]))   # totals < 2^33: exact
    n_ref, n_used, n_fwd = (int(v) for v in host[:3].tolist())
    align = _align(host[3:].view(3, 4)).to(images.device)
    if layout == "glb":
        pos, cols, idx = mesher.compact(points.view(-1, 3), n_used, n_fwd)
        return {"positions": pos, "colors": cols, "indices": idx, "conf_threshold": thr, "align": align}
    faces, face_colors = mesher.faces(n_ref)
    return {"vertices": points.view(-1, 3).clone(), "face_colors": face_colors, "faces": faces, "conf_threshold": thr,
            "align": align}
