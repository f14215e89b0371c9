"""A predictions dict on the device: its cameras and world points (``postprocess``), and the sky, point cloud, mesh,
fused mesh, matches and tracks of one scene, the bundle adjustment of those tracks, and the scores of a scene against its
ground truth.  They read no weight; ``OmniVGGT`` exposes each
under the same name.  Each checks its arguments before any library call (``_check_views``), then takes the scene's views
from ``_kept_views``."""
from __future__ import annotations

import math
import numbers
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


_TRACK_KEYS = (("points", torch.float64, ("n", 3)), ("colors", torch.uint8, ("n", 3)), ("error", torch.float64, ("n",)),
               ("offsets", torch.int64, ("n1",)), ("view", torch.int32, ("m",)), ("xy", torch.int64, ("m", 2)),
               ("point2d", torch.int32, ("m",)), ("view_offsets", torch.int64, ("V1",)), ("view_track", torch.int32, ("m",)),
               ("view_xy", torch.int64, ("m", 2)), ("extrinsic", torch.float32, ("V", 3, 4)),
               ("intrinsic", torch.float32, ("V", 3, 3)))


def _check_tracks(tracks) -> None:
    """ValueError unless ``tracks`` has the keys, dtypes, shapes and one device of what ``tracks`` returns."""
    if not isinstance(tracks, dict) or any(not torch.is_tensor(tracks.get(k)) for k, _, _ in _TRACK_KEYS):
        raise ValueError("bundle_adjust needs the dict tracks() returns")
    n, m, V = tracks["points"].shape[0], tracks["view"].shape[0], tracks["extrinsic"].shape[0]
    sizes = {"n": n, "n1": n + 1, "m": m, "V": V, "V1": V + 1}
    dev = tracks["points"].device
    for k, dtype, shape in _TRACK_KEYS:
        t = tracks[k]
        want = tuple(sizes.get(d, d) for d in shape)
        if t.dtype != dtype or tuple(t.shape) != want or t.device != dev:
            raise ValueError(f"tracks[{k!r}]: expected {dtype} {want} on device {dev}, got {t.dtype} {tuple(t.shape)} on device "
                             f"{t.device}")


@torch.no_grad()
def bundle_adjust(tracks: Dict[str, torch.Tensor], *, iterations: int = 100, refine_focal: bool = True,
                  loss: str = "trivial", loss_scale: float = 1.0) -> Dict[str, object]:
    """Bundle adjustment of the output of ``tracks`` on the device (libovg ovg_bundle_adjust); no counterpart in the reference.

    COLMAP's default PINHOLE bundle adjustment: the residual of an observation is ``tracks``' error formula, (fx X/Z + cx +
    0.5 - (x + 0.5), fy Y/Z + cy + 0.5 - (y + 0.5)) with (X, Y, Z) = R P + t, and the cost is 1/2 sum rho(|r|^2), rho(s) = s
    (``loss="trivial"``) or c^2 log(1 + s/c^2) with c = ``loss_scale`` pixels (``"cauchy"``).  Robust losses weight the
    normal equations by rho'(s) (IRLS) without Ceres' second-order correction: the minimiser is the same, the path to it may
    differ.  Refined: every view's rotation and translation, fx and fy when ``refine_focal`` (the principal point stays), and
    every track point.  The gauge keeps the predictions' frame and scale: view 0's pose and the largest coordinate of view 1's
    baseline t1 - R1 R0^T t0 are held.  Tracks with one observation or seen behind a camera (``error`` +inf) are held and
    left out of the cost.  Levenberg-Marquardt with a Schur complement and preconditioned conjugate gradients, at most
    ``iterations`` steps; the rules are in include/ovg.h and INTEGRATION.md ("Bundle adjustment").

    Returns a new dict with the keys of ``tracks``: ``points`` fp64 [n, 3], ``extrinsic`` fp64 [V, 3, 4] and ``intrinsic``
    fp64 [V, 3, 3] refined, ``error`` recomputed with them, the other tensors of ``tracks`` as they are, and ``ba``: ``cost``
    fp64 [2] (initial and final 1/2 sum rho), ``steps``, ``accepted`` and ``pcg_iterations`` int64, ``status`` int32 (0
    converged, 1 ``iterations`` reached, 2 the trust region collapsed, 3 nothing to refine), all on the device.  No host read."""
    if not geometry._is_int(iterations) or not 1 <= iterations <= 2 ** 31 - 1:
        raise ValueError(f"iterations must be an integer in [1, 2^31 - 1], got {iterations!r}")
    if loss not in ops.BA_LOSSES:
        raise ValueError(f"loss must be 'trivial' or 'cauchy', got {loss!r}")
    if not (isinstance(loss_scale, numbers.Real) and not isinstance(loss_scale, bool) and math.isfinite(loss_scale)
            and loss_scale > 0):
        raise ValueError(f"loss_scale must be a finite number > 0, got {loss_scale!r}")
    _check_tracks(tracks)
    V = tracks["extrinsic"].shape[0]
    if not 2 <= V <= 256:
        raise ValueError(f"bundle_adjust needs 2 to 256 views, got {V}")
    obs = tracks["xy"].to(torch.float64) + 0.5                           # COLMAP's pixel centres
    points, ext, intr, error, cost, stats = ops.bundle_adjust(
        tracks["points"].contiguous(), tracks["offsets"].contiguous(), tracks["view"].contiguous(), obs,
        tracks["extrinsic"].contiguous(), tracks["intrinsic"].contiguous(), iterations=iterations,
        refine_focal=refine_focal, loss=loss, loss_scale=loss_scale)
    out = dict(tracks)
    out.update(points=points, extrinsic=ext, intrinsic=intr, error=error,
               ba={"cost": cost, "steps": stats[0], "accepted": stats[1], "pcg_iterations": stats[2],
                   "status": stats[3].to(torch.int32)})
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


def _fusion_grid(lo: np.ndarray, hi: np.ndarray, resolution: int):
    """(origin fp32 [3], voxel fp32, trunc fp32, (nz, ny, nx)) from the kept points' 1st / 99th percentiles, in fp64 on the
    host; None for a zero extent."""
    L = float((hi - lo).max())
    if not L > 0:
        return None
    margin = 0.05 * L
    s = np.float32((L + 2 * margin) / resolution)
    origin = (lo - margin).astype(np.float32)
    n = [min(math.ceil((hi[a] - lo[a] + 2 * margin) / float(s)) + 1, resolution + 1) for a in range(3)]
    return origin, s, np.float32(4.0 * float(s)), (n[2], n[1], n[0])


def _fusion(predictions, resolution, conf_percent, conf_floor, scene, mask_sky):
    """fused_mesh, and the volume it extracted from: (result, tsdf, color), both volumes None when the result is empty."""
    _check_views(predictions, "depth", conf_percent, conf_floor, None, scene, mask_sky)
    if not geometry._is_int(resolution) or not 16 <= resolution <= 512:
        raise ValueError(f"resolution must be an integer in [16, 512], got {resolution!r}")
    if "depth" not in predictions:
        raise ValueError("fused_mesh needs the predictions' depth")
    if not ("extrinsic" in predictions and "intrinsic" in predictions or "pose_enc" in predictions):
        raise ValueError("fused_mesh needs extrinsic and intrinsic, or pose_enc to decode them from")
    S = _of_scene(predictions["images"], 3, scene).shape[0]
    H, W = predictions["images"].shape[-2:]
    if S * H * W >= 2 ** 31:
        raise ValueError(f"fused_mesh needs views * H * W < 2^31, got {S} x {H} x {W}")
    images, (ext, intr), points, mask, thr, _ = _kept_views(predictions, "depth", conf_percent, conf_floor, None, scene,
                                                           mask_sky, cameras="predictions")
    dev = images.device
    host = ops.host_read(torch.cat([ops.tsdf_bounds(points, mask), ext[0].double().reshape(-1)]))
    if host[7]:
        raise ValueError("kept points must be finite (cKDTree: data must be finite, check for nan or inf values)")
    align = _align(host[8:].view(3, 4)).to(dev)
    lo, hi = host[1:4].numpy(), host[4:7].numpy()
    grid = _fusion_grid(lo, hi, resolution) if host[0] > 0 else None
    out = {"positions": torch.empty(0, 3, device=dev), "colors": torch.empty(0, 3, device=dev, dtype=torch.uint8),
           "indices": torch.empty(0, 3, device=dev, dtype=torch.int32), "conf_threshold": thr, "align": align,
           "origin": torch.zeros(3, device=dev), "voxel_size": torch.zeros((), device=dev)}
    if grid is None:
        return out, None, None
    origin, s, trunc, shape = grid
    ws = ops.tsdf_workspace(dev, shape)
    depth = _of_scene(predictions["depth"], 3, scene).float().reshape(S, H, W).contiguous()
    tsdf, color = ops.tsdf_integrate(depth, mask, images, ext, intr, shape, origin, s, trunc, ws)
    mc = ops.TsdfMesher(tsdf, origin, s, ws)
    m, k = (int(v) for v in ops.host_read(mc.totals).tolist())
    out.update(origin=torch.from_numpy(origin).to(dev), voxel_size=torch.tensor(s, device=dev))
    if k:
        out["positions"], out["colors"], out["indices"] = mc.extract(color, m, k)
    return out, tsdf, color


@torch.no_grad()
def fused_mesh(predictions: Dict[str, object], *, resolution: int = 512, conf_percent: float = 50.0,
               conf_floor: float = 1e-5, scene: int = 0, mask_sky=False) -> Dict[str, torch.Tensor]:
    """One coloured surface of a scene: its depth maps fused into a truncated signed distance (TSDF) volume and the volume's
    zero level set extracted by marching cubes, on the device (libovg ovg_tsdf_*); no counterpart in the reference.  Where
    ``mesh`` gives every view its own sheet of triangles, each surface seen by several views appears once here.

    Kept pixels are ``point_cloud``'s with ``source="depth"`` (``conf_percent``, ``conf_floor``, ``mask_sky``); the cameras are
    the predictions' ``extrinsic`` / ``intrinsic``, decoded from ``pose_enc`` where missing, as ``tracks`` takes them.
    Grid: per axis lo / hi = numpy.percentile(kept points, 1 / 99), L = max(hi - lo), margin = 0.05 L, voxel s = (L + 2 margin)
    / ``resolution`` (an integer in [16, 512]), at most resolution + 1 voxels per axis, truncation 4 s.  Only the 8^3-voxel
    bricks that some kept pixel's band d -/+ 4 s touches are integrated; a voxel's value is the mean over the views that see
    it in front of the truncation band of min(1, (d - z) / 4 s), its colour the mean colour of those pixels.  Triangles face
    the free space (the cameras).  The rules are in include/ovg.h and INTEGRATION.md ("Fused mesh").

    Returns on the device ``positions`` fp32 [m, 3], ``colors`` uint8 [m, 3] and ``indices`` int32 [k, 3] for
    ``glb.write_mesh_glb``, ``conf_threshold`` and ``align`` as ``point_cloud`` returns them, and the grid: ``origin`` fp32 [3]
    (voxel (0, 0, 0)) and ``voxel_size`` (0-d fp32).  No kept pixel or a zero extent gives an empty mesh (origin 0, voxel
    size 0).  Two host reads: the bounds with the first camera, then the mesh's sizes.  Kept points that are not finite raise
    ValueError."""
    return _fusion(predictions, resolution, conf_percent, conf_floor, scene, mask_sky)[0]


EVAL_MAX_CAMERA_VIEWS = 8192          # pose group: at most 33.5 M pairs (537 MB of pair errors)
EVAL_MAX_POINT_PIXELS = 2 ** 30       # points group: S H W below the matcher's limit
EVAL_MAX_POINT_VIEWS = 65535          # points group: the unprojection's views


def _gt_tensor(t, name: str, S: int, tail, device, scene: int, alt_tail=None) -> Optional[torch.Tensor]:
    """A ground-truth tensor [B, S, *tail] or [S, *tail] (or *alt_tail) of the scene, checked: None stays None."""
    if t is None:
        return None
    if not torch.is_tensor(t):
        raise ValueError(f"{name} must be a tensor, got {type(t).__name__}")
    shape = tuple(t.shape)
    has_b = None
    for tl in [tuple(tail)] + ([tuple(alt_tail)] if alt_tail is not None else []):
        if shape == (S,) + tl:
            has_b = False
        elif len(shape) == len(tl) + 2 and shape[1:] == (S,) + tl and 0 <= scene < shape[0]:
            has_b = True
    if has_b is None:
        tails = [tail] + ([alt_tail] if alt_tail is not None else [])
        want = " or ".join(f"[B, {S}, {', '.join(map(str, tl))}] / [{S}, {', '.join(map(str, tl))}]" for tl in tails)
        raise ValueError(f"{name} must have shape {want}, got {list(shape)}")
    allowed = (torch.bool, torch.uint8) if name == "mask" else ()
    if not (t.dtype.is_floating_point or t.dtype in allowed):
        raise ValueError(f"{name} must be a floating tensor{' (or bool / uint8)' if allowed else ''}, got {t.dtype}")
    if t.device != device:
        raise ValueError(f"{name} is on {t.device}, the predictions on {device}")
    return t[scene] if has_b else t


def _check_eval_views(views, S: int) -> List[int]:
    """The scored views, ascending: every view when None, else distinct integers in [0, S)."""
    if views is None:
        return list(range(S))
    views = list(views)
    if not all(geometry._is_int(v) for v in views):
        raise ValueError(f"views must be integers, got {views!r}")
    if any(not 0 <= v < S for v in views):
        raise ValueError(f"views must be in [0, {S}), got {views!r}")
    if len(set(int(v) for v in views)) != len(views):
        raise ValueError(f"views must not repeat, got {views!r}")
    if not views:
        raise ValueError("views must not be empty")
    return sorted(int(v) for v in views)


@torch.no_grad()
def evaluate(predictions: Dict[str, object], *, extrinsics=None, intrinsics=None, depth=None, mask=None, views=None,
             source: str = "depth", scene: int = 0) -> Dict[str, Dict[str, torch.Tensor]]:
    """Scores of one scene's predictions against its ground truth, on the device (libovg ovg_eval_*).  The reference scores
    trajectories only, on the host through evo (vo_eval.py:163-246 eval_metrics); the definitions are in include/ovg.h and
    INTEGRATION.md ("Evaluation").

    Ground truth in the layout ``preprocess.load_images_and_cameras`` returns and the forward takes, with or without B:
    ``extrinsics`` world-to-camera [B, S, 3, 4] / [B, S, 4, 4], ``intrinsics`` [B, S, 3, 3], ``depth`` [B, S, H, W(, 1)] at
    the model's resolution, ``mask`` [B, S, H, W] (non-zero: valid; default every pixel).  A view has a ground-truth camera
    when fx, fy > 0 and its extrinsic is finite (the loader's zero placeholders have none); a pixel has ground-truth depth
    when its mask is set and the depth is > 0 and finite.  ``views`` (default: all) restricts every metric to those views,
    e.g. the ones whose ground truth did not go into the forward.

    Predictions: cameras ``extrinsic`` (decoded from ``pose_enc`` where missing, as ``tracks`` takes them), depth ``depth``,
    points ``world_points_from_depth`` (``source="depth"``; unprojected through the decoded cameras when missing) or
    ``world_points`` (``"pointmap"``).  A group is computed when its ground truth is given:
      "pose" (extrinsics and intrinsics): ``ate``, ``rpe_trans``, ``rpe_rot`` (evo's APE / RPE after the Umeyama Sim(3) of
          the camera centres, as vo_eval.py:190-236), ``auc`` / ``rra`` / ``rta`` fp64 [3] at 5, 10, 30 degrees (the
          pairwise protocol of the VGGT family), ``sim3`` fp64 [4, 4], ``views`` (the count n), ``pairs`` int32 [P, 2],
          ``pair_errors`` fp64 [P, 2] (RRE, RTE in degrees), ``rpe_errors`` fp64 [n - 1, 2] (|t|, degrees).
      "depth" (depth): ``abs_rel``, ``sq_rel``, ``rmse``, ``delta`` fp64 [3] after per-scene median scaling ``scale``, with
          ``pixels``, ``view_abs_rel``, ``view_delta1``, ``view_pixels`` [S].  No valid pixel gives NaN and 0 pixels.
      "points" (depth and cameras): ``acc``, ``acc_median``, ``comp``, ``comp_median``, ``chamfer`` (nearest-neighbour
          distances between the Umeyama-aligned prediction and the ground-truth points, exact), ``nc_acc``, ``nc_comp``, ``nc``
          (normal consistency with grid normals, not Open3D's k-NN normals), ``pixels``, ``sim3``, ``acc_dist`` /
          ``comp_dist`` fp64 [pixels].
    Every value is a device tensor.  Host reads: the pose fit's status (``ovg_eval_pose``), the point fit's status
    (``ovg_sim3_estimate``) and the matcher's non-finite flag (``ovg_match_query``): at most three.  ValueError before any
    device work for wrong shapes or dtypes, bad ``views``, ``source="pointmap"`` without ``world_points``, no ground truth,
    more than 8192 scored views with cameras, S H W >= 2^31, and, when both cameras and depth are given (the points group),
    S H W >= 2^30 or S > 65535 views; after a read, for fewer than 3 views or pixels to align, or collinear ones.  S H W need
    not be a multiple of 4, and the ground truth may be a view at any storage offset."""
    if source not in ("depth", "pointmap"):
        raise ValueError(f"source must be 'depth' or 'pointmap', got {source!r}")
    images = predictions["images"]
    S, _, H, W = _of_scene(images, 3, scene).shape
    dev = images.device
    if S * H * W >= 2 ** 31:
        raise ValueError(f"evaluate needs views * H * W < 2^31, got {S} x {H} x {W}")
    gext = _gt_tensor(extrinsics, "extrinsics", S, (3, 4), dev, scene, alt_tail=(4, 4))
    gint = _gt_tensor(intrinsics, "intrinsics", S, (3, 3), dev, scene)
    gdep = _gt_tensor(depth, "depth", S, (H, W), dev, scene, alt_tail=(H, W, 1))
    gmask = _gt_tensor(mask, "mask", S, (H, W), dev, scene)
    if (gext is None) != (gint is None):
        raise ValueError("ground-truth cameras need both extrinsics and intrinsics")
    cams = gext is not None
    if not cams and gdep is None:
        raise ValueError("evaluate needs ground truth: extrinsics and intrinsics, depth, or both")
    if gmask is not None and gdep is None:
        raise ValueError("mask needs depth")
    sel = _check_eval_views(views, S)
    if cams and len(sel) > EVAL_MAX_CAMERA_VIEWS:
        raise ValueError(f"the pose group scores at most {EVAL_MAX_CAMERA_VIEWS} views, got {len(sel)}")
    if cams and not ("extrinsic" in predictions or "pose_enc" in predictions):
        raise ValueError("the pose group needs the predictions' extrinsic, or pose_enc to decode it from")
    if gdep is not None and "depth" not in predictions:
        raise ValueError("the depth group needs the predictions' depth")
    if cams and gdep is not None:
        if S * H * W >= EVAL_MAX_POINT_PIXELS or S > EVAL_MAX_POINT_VIEWS:
            raise ValueError(f"the points group needs views * H * W < 2^30 and at most {EVAL_MAX_POINT_VIEWS} views, got "
                             f"{S} x {H} x {W}")
        if source == "pointmap" and "world_points" not in predictions:
            raise ValueError("source='pointmap' needs the predictions' world_points")
        if source == "depth" and "world_points_from_depth" not in predictions and "pose_enc" not in predictions:
            raise ValueError("source='depth' needs world_points_from_depth, or pose_enc and depth to compute it")

    out: Dict[str, Dict[str, torch.Tensor]] = {}
    hw = H * W
    view_sel = torch.zeros(S, dtype=torch.uint8)
    view_sel[sel] = 1
    view_sel = view_sel.to(dev)
    if cams:
        gext = gext[..., :3, :4].float().contiguous()
        gint = gint.float().contiguous()
        if "extrinsic" in predictions:
            pext = _of_scene(predictions["extrinsic"], 2, scene).float().contiguous()
        else:
            pext, _, _ = decode_cameras(_of_scene(predictions["pose_enc"], 1, scene), None, H, W)
        sim3, stats, pairs, perr, rpe, sc = ops.eval_pose(gext, gint, pext, torch.tensor(sel, dtype=torch.int32).to(dev))
        n_views, status = (int(v) for v in ops.host_read(stats[:2]).tolist())
        if status:
            raise ValueError(f"evaluate: the pose alignment is degenerate: {geometry.SIM3_STATUS[status]}")
        P = n_views * (n_views - 1) // 2
        out["pose"] = {"ate": sc[0], "rpe_trans": sc[1], "rpe_rot": sc[2], "auc": sc[3:6], "rra": sc[6:9], "rta": sc[9:12],
                       "sim3": sim3, "views": stats[0].long(), "pairs": pairs[:P], "pair_errors": perr[:P],
                       "rpe_errors": rpe[:n_views - 1]}
    if gdep is not None:
        gd = gdep.float().reshape(S, hw).contiguous()
        pd = _of_scene(predictions["depth"], 3, scene).float().reshape(S, hw).contiguous()
        m8 = None if gmask is None else (gmask != 0).to(torch.uint8).reshape(S, hw).contiguous()
        sc, var, vd1, vpix = ops.eval_depth(gd, m8, pd, view_sel)
        out["depth"] = {"pixels": sc[0].long(), "scale": sc[1], "median_gt": sc[2], "median_pred": sc[3], "abs_rel": sc[4],
                        "sq_rel": sc[5], "rmse": sc[6], "delta": sc[7:10], "view_abs_rel": var, "view_delta1": vd1,
                        "view_pixels": vpix}
    if cams and gdep is not None:
        if source == "pointmap":
            pts = _of_scene(predictions["world_points"], 3, scene)
        elif "world_points_from_depth" in predictions:
            pts = _of_scene(predictions["world_points_from_depth"], 3, scene)
        else:
            _, _, pts = decode_cameras(_of_scene(predictions["pose_enc"], 1, scene), _of_scene(predictions["depth"], 3, scene),
                                       H, W)
        pts = pts.float().reshape(S, hw, 3).contiguous()
        c2w, keep = ops.eval_points_keep(gext, gint, gd, m8, pts, view_sel)
        clouds = torch.empty(2, S * hw, 3, device=dev, dtype=torch.float32)
        # ovg_unproject_depth wants 16-byte aligned depth and points: a depth view at an odd offset is copied, and when S H W
        # is not a multiple of 4 (clouds[1] starts S H W 12 bytes in) the points go through a fresh tensor (same values)
        gdu = gd if gd.data_ptr() % 16 == 0 else gd.clone()
        if clouds[1].data_ptr() % 16 == 0:
            ops.unproject_depth(gdu.view(S, H, W), gint, c2w, H, W, out=clouds[1])
        else:
            clouds[1].copy_(ops.unproject_depth(gdu.view(S, H, W), gint, c2w, H, W).view(S * hw, 3))
        sim3p, stp = ops.sim3_estimate(pts.view(-1, 3), clouds[1], keep[0])
        n_pix, status = (int(v) for v in ops.host_read(stp[:2]).tolist())
        if status:
            raise ValueError(f"evaluate: the point alignment is degenerate: {geometry.SIM3_STATUS[status]}")
        ops.sim3_apply(sim3p, S, hw, points=((pts.view(-1, 3), clouds[0]),))
        mt = ops.Matcher(clouds, keep, torch.tensor([[0, 1]], dtype=torch.int32).to(dev))
        _, nonfinite = mt.counts()
        if nonfinite:
            raise ValueError("evaluate: an aligned or ground-truth point is not finite")
        acc, comp, sc = ops.eval_points(mt, S, H, W)
        out["points"] = {"pixels": sc[0].long(), "acc": sc[1], "acc_median": sc[2], "comp": sc[3], "comp_median": sc[4],
                         "chamfer": sc[5], "nc_acc": sc[6], "nc_comp": sc[7], "nc": sc[8], "sim3": sim3p,
                         "acc_dist": acc[:n_pix], "comp_dist": comp[:n_pix]}
    return out
