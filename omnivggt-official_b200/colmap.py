"""COLMAP sparse-model export of ``OmniVGGT.tracks`` (host code): ``cameras``, ``images`` and ``points3D`` in COLMAP's binary
or text layout (its documented read_write_model formats), plus the model-resolution images, so the folder is a dataset
that COLMAP, glomap, nerfstudio's COLMAP importer and Gaussian-splatting trainers read as it is.

Conventions: one PINHOLE camera per view (the predicted intrinsics differ per view), ``camera_id = image_id = view + 1`` and
``point3D_id = track + 1``.  The reference unprojects pixel index (x, y) through ((x - cx) / fx, (y - cy) / fy)
(utils/geometry.py:236-264), while COLMAP puts the centre of pixel (x, y) at (x + 0.5, y + 0.5): the cameras store
(fx, fy, cx + 0.5, cy + 0.5) and the observations (x + 0.5, y + 0.5).  The image pose is the world-to-camera ``extrinsic``:
tvec = t and qvec = (w, x, y, z) of R by the reference's mat_to_quat (utils/rotation.py:47-109), in fp64."""
from __future__ import annotations

import os
from typing import Dict, Optional, Sequence

import numpy as np

PINHOLE = 1                     # COLMAP's model id

_CAMERA = np.dtype([("camera_id", "<i4"), ("model_id", "<i4"), ("width", "<u8"), ("height", "<u8"), ("params", "<f8", 4)])
_IMAGE = np.dtype([("image_id", "<i4"), ("qvec", "<f8", 4), ("tvec", "<f8", 3), ("camera_id", "<i4")])
_POINT2D = np.dtype([("xy", "<f8", 2), ("point3D_id", "<i8")])
_POINT3D = np.dtype([("point3D_id", "<u8"), ("xyz", "<f8", 3), ("rgb", "u1", 3), ("error", "<f8"), ("track_length", "<u8")])
_TRACK = np.dtype([("image_id", "<i4"), ("point2D_idx", "<i4")])


def rotmat_to_qvec(R: np.ndarray) -> np.ndarray:
    """COLMAP qvec (w, x, y, z) fp64 [..., 4] of rotation matrices R [..., 3, 3]: the reference's mat_to_quat evaluated in
    fp64 (the best-conditioned of the four candidates, real part made non-negative), reordered from (x, y, z, w)."""
    R = np.asarray(R, np.float64)
    m = R.reshape(R.shape[:-2] + (9,))
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = (m[..., i] for i in range(9))
    arg = np.stack([1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22, 1.0 - m00 - m11 + m22], -1)
    q_abs = np.where(arg > 0, np.sqrt(np.maximum(arg, 0.0)), 0.0)
    rijk = np.stack([np.stack([q_abs[..., 0] ** 2, m21 - m12, m02 - m20, m10 - m01], -1),
                     np.stack([m21 - m12, q_abs[..., 1] ** 2, m10 + m01, m02 + m20], -1),
                     np.stack([m02 - m20, m10 + m01, q_abs[..., 2] ** 2, m12 + m21], -1),
                     np.stack([m10 - m01, m20 + m02, m21 + m12, q_abs[..., 3] ** 2], -1)], -2)
    cand = rijk / (2.0 * np.maximum(q_abs, 0.1)[..., None])
    best = np.take_along_axis(cand, np.argmax(q_abs, -1)[..., None, None], -2)[..., 0, :]    # (r, i, j, k)
    return np.where(best[..., :1] < 0, -best, best)


def _check_names(names: Sequence[str], V: int):
    names = [str(n) for n in names]
    if len(names) != V:
        raise ValueError(f"image_names must hold one name per view ({V}), got {len(names)}")
    if len(set(names)) != V:
        raise ValueError("image_names must be unique")
    for n in names:
        if not n or "/" in n or "\\" in n or os.sep in n or "\0" in n or n in (".", ".."):
            raise ValueError(f"an image name is a plain file name, got {n!r}")
    return names


def _scatter(buf: np.ndarray, pos: np.ndarray, rows: np.ndarray, chunk: int = 1 << 16):
    """buf[pos[i] : pos[i] + w] = rows[i] for byte rows [k, w], in chunks so the index arrays stay small."""
    col = np.arange(rows.shape[1], dtype=np.int64)
    for s in range(0, len(rows), chunk):
        buf[pos[s:s + chunk, None] + col] = rows[s:s + chunk]


def _model(predictions: Dict[str, object], tracks: Dict[str, object], scene: int):
    """The model as host numpy arrays."""
    def host(t):
        return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)

    images = predictions["images"]
    images = host(images[scene] if images.dim() == 5 else images)
    t = {k: host(v) for k, v in tracks.items()}
    V, _, H, W = images.shape
    if t["view_offsets"].shape != (V + 1,) or t["extrinsic"].shape != (V, 3, 4) or t["intrinsic"].shape != (V, 3, 3):
        raise ValueError("the tracks do not belong to this scene's views")
    return images, t


def write_colmap(path: str, predictions: Dict[str, object], tracks: Dict[str, object], *,
                 image_names: Optional[Sequence[str]] = None, images: bool = True, binary: bool = True, scene: int = 0) -> str:
    """Writes ``path/sparse/0/{cameras,images,points3D}.bin`` (``.txt`` with ``binary=False``) from ``OmniVGGT.tracks``'s
    result, and with ``images`` the model-resolution images ``path/images/<name>`` as PNG, so image sizes match the
    cameras.  ``image_names`` (default ``f"{i:06d}.png"``): V unique plain file names.  Each image's POINTS2D are its
    observations in row-major pixel order, every one in a track.  Text floats are ``repr``, so they parse back to the same
    doubles.  Returns the sparse model's directory."""
    imgs, t = _model(predictions, tracks, scene)
    V, _, H, W = imgs.shape
    names = _check_names(image_names if image_names is not None else [f"{i:06d}.png" for i in range(V)], V)
    sparse = os.path.join(path, "sparse", "0")
    os.makedirs(sparse, exist_ok=True)

    K, E = t["intrinsic"].astype(np.float64), t["extrinsic"].astype(np.float64)
    cams = np.zeros(V, _CAMERA)
    cams["camera_id"] = np.arange(1, V + 1)
    cams["model_id"] = PINHOLE
    cams["width"], cams["height"] = W, H
    cams["params"] = np.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2] + 0.5, K[:, 1, 2] + 0.5], 1)
    ims = np.zeros(V, _IMAGE)
    ims["image_id"] = ims["camera_id"] = np.arange(1, V + 1)
    ims["qvec"] = rotmat_to_qvec(E[:, :, :3])
    ims["tvec"] = E[:, :, 3]
    vo = t["view_offsets"]
    p2d = np.zeros(len(t["view_track"]), _POINT2D)
    p2d["xy"] = t["view_xy"] + 0.5
    p2d["point3D_id"] = t["view_track"].astype(np.int64) + 1
    n, m = len(t["points"]), len(t["view"])
    p3d = np.zeros(n, _POINT3D)
    p3d["point3D_id"] = np.arange(1, n + 1)
    p3d["xyz"], p3d["rgb"], p3d["error"] = t["points"], t["colors"], t["error"]
    p3d["track_length"] = np.diff(t["offsets"])
    trk = np.zeros(m, _TRACK)
    trk["image_id"] = t["view"] + 1
    trk["point2D_idx"] = t["point2d"]

    if binary:
        with open(os.path.join(sparse, "cameras.bin"), "wb") as f:
            f.write(np.uint64(V).astype("<u8").tobytes() + cams.tobytes())
        with open(os.path.join(sparse, "images.bin"), "wb") as f:
            f.write(np.uint64(V).astype("<u8").tobytes())
            for i in range(V):
                f.write(ims[i:i + 1].tobytes() + names[i].encode() + b"\0"
                        + np.uint64(vo[i + 1] - vo[i]).astype("<u8").tobytes() + p2d[vo[i]:vo[i + 1]].tobytes())
        # record of track k at 8 + 51 k + 8 offsets[k] (51-byte header, 8 bytes per observation)
        buf = np.empty(8 + _POINT3D.itemsize * n + _TRACK.itemsize * m, np.uint8)
        buf[:8] = np.frombuffer(np.uint64(n).astype("<u8").tobytes(), np.uint8)
        start = 8 + _POINT3D.itemsize * np.arange(n, dtype=np.int64) + _TRACK.itemsize * t["offsets"][:-1]
        _scatter(buf, start, p3d.view(np.uint8).reshape(n, _POINT3D.itemsize))
        owner = np.repeat(np.arange(n, dtype=np.int64), np.diff(t["offsets"]))
        obs_at = 8 + _POINT3D.itemsize * (owner + 1) + _TRACK.itemsize * np.arange(m, dtype=np.int64)
        _scatter(buf, obs_at, trk.view(np.uint8).reshape(m, _TRACK.itemsize))
        with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
            f.write(buf.tobytes())
    else:
        _write_text(sparse, V, names, cams, ims, p2d, vo, p3d, trk, t["offsets"])

    if images:
        from PIL import Image
        folder = os.path.join(path, "images")
        os.makedirs(folder, exist_ok=True)
        u8 = (imgs * np.float32(255)).astype(np.uint8).transpose(0, 2, 3, 1)          # the point cloud's colour rule
        for i in range(V):
            Image.fromarray(np.ascontiguousarray(u8[i])).save(os.path.join(folder, names[i]), format="PNG")
    return sparse


def _words(a: np.ndarray) -> np.ndarray:
    """Every element of a as its text: repr for floats (round-trips), str for integers."""
    return np.array([repr(v) for v in a.ravel().tolist()], dtype=object).reshape(a.shape)


def _write_text(sparse, V, names, cams, ims, p2d, vo, p3d, trk, offsets):
    cam_lines = [f"{c} PINHOLE {w} {h} " + " ".join(p) for c, w, h, p in
                 zip(cams["camera_id"].tolist(), cams["width"].tolist(), cams["height"].tolist(), _words(cams["params"]))]
    with open(os.path.join(sparse, "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n"
                f"# Number of cameras: {V}\n" + "".join(line + "\n" for line in cam_lines))
    pose = _words(np.concatenate([ims["qvec"], ims["tvec"]], 1))
    p2w = np.concatenate([_words(p2d["xy"]), _words(p2d["point3D_id"][:, None])], 1)
    mean_obs = float(vo[-1]) / V
    with open(os.path.join(sparse, "images.txt"), "w") as f:
        f.write("# Image list with two lines of data per image:\n"
                "#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n#   POINTS2D[] as (X, Y, POINT3D_ID)\n"
                f"# Number of images: {V}, mean observations per image: {mean_obs!r}\n")
        for i in range(V):
            f.write(f"{i + 1} " + " ".join(pose[i]) + f" {i + 1} {names[i]}\n" + " ".join(p2w[vo[i]:vo[i + 1]].ravel()) + "\n")
    n = len(p3d)
    head = np.concatenate([_words(p3d["point3D_id"][:, None]), _words(p3d["xyz"]), _words(p3d["rgb"].astype(np.int64)),
                           _words(p3d["error"][:, None])], 1)
    tw = np.concatenate([_words(trk["image_id"][:, None]), _words(trk["point2D_idx"][:, None])], 1)
    mean_len = float(offsets[-1]) / n if n else 0.0
    with open(os.path.join(sparse, "points3D.txt"), "w") as f:
        f.write("# 3D point list with one line of data per point:\n"
                "#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n"
                f"# Number of points: {n}, mean track length: {mean_len!r}\n")
        f.writelines(" ".join(head[k]) + " " + " ".join(tw[offsets[k]:offsets[k + 1]].ravel()) + "\n" for k in range(n))
