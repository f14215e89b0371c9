"""numpy restatement of OmniVGGT.tracks (star tracks over reciprocal matches) and of its COLMAP conventions, plus a COLMAP
sparse-model reader and writer written from COLMAP's documented read_write_model layouts, for the tests.

Star tracks, under the contract libovg's ovg_tracks_* implement:
  - node (v, k) = kept point k of view v (kept points in row-major pixel order); the edges are the reciprocal matches of the
    requested pairs, (i, j) and (j, i) being one pair;
  - views anchor in order a = 0 .. V-1; every unclaimed node (a, k) gathers its partners, the reciprocal match of k in each
    view j > a of a pair (a, j) that is unclaimed too; with 1 + partners >= min_views they form a new track and are claimed;
  - tracks in (anchor view, anchor k) order, observations in ascending view order;
  - position: the fp64 sum of the observations' fp32 points in observation order, divided once by the count;
  - colour: the anchor pixel's (image * 255).astype(uint8);
  - error: the mean over the observations of |project(position) - (x + 0.5, y + 0.5)|, every fp64 operation rounded on its
    own: (X, Y, Z) = ((r0 px + r1 py) + r2 pz) + t per row, u = fx (X / Z) + (cx + 0.5), v = fy (Y / Z) + (cy + 0.5);
    +inf when some observation has Z <= 0."""
from __future__ import annotations

import os
import struct

import numpy as np

from oracle import matches_oracle as MO


def normalize_pairs(pairs, V: int) -> np.ndarray:
    """(min, max) of every pair, duplicates merged, sorted: int [P, 2]; all i < j when pairs is None."""
    if pairs is None:
        pairs = [(i, j) for i in range(V) for j in range(i + 1, V)]
    p = np.sort(np.asarray(list(pairs), np.int64).reshape(-1, 2), axis=1)
    return np.unique(p, axis=0).reshape(-1, 2)


def pair_matches(pts_kept, pairs, nn=MO.nn_brute):
    """{(i, j): (k_i, k_j)}: the reciprocal matches of every normalised pair in kept-index space, by matches_oracle."""
    out = {}
    for i, j in pairs:
        rec, nn2, _ = MO.find_reciprocal_matches(pts_kept[i], pts_kept[j], nn)
        kj = np.flatnonzero(rec)
        out[(int(i), int(j))] = (nn2[rec].astype(np.int64), kj.astype(np.int64))
    return out


def star_tracks(n_kept, matches, min_views: int):
    """The star rule on a match graph.  n_kept: kept nodes per view; matches: {(i, j): (k_i, k_j)} with i < j and a
    one-to-one matching per pair.  Returns (offsets int64 [n + 1], obs_view int64 [m], obs_k int64 [m])."""
    V = len(n_kept)
    claim = [np.full(n, -1, np.int64) for n in n_kept]
    n_tracks = 0
    rows_v, rows_k = [], []                        # per step: member matrices [n_new, 1 + partner views], -1 = absent
    for a in range(V):
        cand = np.flatnonzero(claim[a] < 0)
        views, cols = [a], [cand]
        for j in sorted(j for (i, j) in matches if i == a):
            ki, kj = matches[(a, j)]
            partner = np.full(n_kept[a], -1, np.int64)
            partner[ki] = kj
            pk = partner[cand]
            ok = pk >= 0
            ok[ok] = claim[j][pk[ok]] < 0
            views.append(j)
            cols.append(np.where(ok, pk, -1))
        mk = np.stack(cols, 1)
        mk = mk[(mk >= 0).sum(1) >= min_views]
        ids = n_tracks + np.arange(len(mk))
        for c, v in enumerate(views):
            there = mk[:, c] >= 0
            claim[v][mk[there, c]] = ids[there]
        n_tracks += len(mk)
        rows_v.append(np.where(mk >= 0, np.asarray(views)[None, :], -1))
        rows_k.append(mk)
    lengths = np.concatenate([(mk >= 0).sum(1) for mk in rows_k]) if rows_k else np.zeros(0, np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    obs_v = np.concatenate([mv[mk >= 0] for mv, mk in zip(rows_v, rows_k)]).astype(np.int64)   # row-major: track, view
    obs_k = np.concatenate([mk[mk >= 0] for mk in rows_k]).astype(np.int64)
    return offsets, obs_v, obs_k


def scene_tracks(points, keep, images, extrinsic, intrinsic, pairs=None, min_views: int = 2, nn=MO.nn_brute, matches=None):
    """The whole of OmniVGGT.tracks on host arrays: points fp32 [V, H, W, 3], keep bool [V, H, W], images fp32 [V, 3, H, W],
    extrinsic [V, 3, 4], intrinsic [V, 3, 3].  matches: given per-pair matches (pair_matches' layout) instead of computing
    them with nn.  Returns the device's dict as numpy arrays."""
    points = np.asarray(points, np.float32)
    V, H, W, _ = points.shape
    flat = points.reshape(V, H * W, 3)
    kp = np.asarray(keep, bool).reshape(V, H * W)
    kept_rows = [np.flatnonzero(kp[v]) for v in range(V)]
    pts_kept = [flat[v][kept_rows[v]] for v in range(V)]
    pairs = normalize_pairs(pairs, V)
    if matches is None:
        matches = pair_matches(pts_kept, pairs, nn)
    offsets, ov, ok = star_tracks([len(r) for r in kept_rows], matches, min_views)
    n, m = len(offsets) - 1, len(ov)
    first = np.concatenate([[0], np.cumsum([len(r) for r in kept_rows])]).astype(np.int64)
    node = first[ov] + ok
    row = np.concatenate(kept_rows).astype(np.int64)[node]
    P = np.concatenate(pts_kept).astype(np.float64)[node]
    length = np.diff(offsets)
    slot = np.arange(m) - np.repeat(offsets[:-1], length)
    owner = np.repeat(np.arange(n), length)
    s = np.zeros((n, 3))
    for c in range(int(length.max()) if n else 0):           # observation order inside every track
        at = slot == c
        s[owner[at]] = s[owner[at]] + P[at]
    cnt = length.astype(np.float64)
    pos = s / cnt[:, None]
    E = np.asarray(extrinsic, np.float32).astype(np.float64)[ov]
    K = np.asarray(intrinsic, np.float32).astype(np.float64)[ov]
    X = pos[owner]
    cam = [((E[:, r, 0] * X[:, 0] + E[:, r, 1] * X[:, 1]) + E[:, r, 2] * X[:, 2]) + E[:, r, 3] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[:, 0, 0] * (cam[0] / cam[2]) + (K[:, 0, 2] + 0.5)
        v = K[:, 1, 1] * (cam[1] / cam[2]) + (K[:, 1, 2] + 0.5)
        du = u - ((row % W).astype(np.float64) + 0.5)
        dv = v - ((row // W).astype(np.float64) + 0.5)
        e = np.sqrt(du * du + dv * dv)
    esum = np.zeros(n)
    for c in range(int(length.max()) if n else 0):
        at = slot == c
        esum[owner[at]] = esum[owner[at]] + e[at]
    behind = np.zeros(n, bool)
    np.logical_or.at(behind, owner, cam[2] <= 0)
    err = np.where(behind, np.inf, esum / cnt)
    img = np.asarray(images, np.float32)
    u8 = (img * np.float32(255)).astype(np.uint8)                      # visual_util.py:202
    anchor = offsets[:-1]
    colors = u8[ov[anchor], :, row[anchor] // W, row[anchor] % W] if n else np.zeros((0, 3), np.uint8)
    xy = np.stack([row % W, row // W], 1) if m else np.zeros((0, 2), np.int64)
    # per view: claimed nodes in row-major order, and each observation's rank there
    order = np.lexsort((row, ov))
    view_offsets = np.concatenate([[0], np.cumsum(np.bincount(ov, minlength=V))]).astype(np.int64)
    point2d = np.empty(m, np.int64)
    point2d[order] = np.arange(m) - view_offsets[ov[order]]
    return {"points": pos, "colors": colors.astype(np.uint8), "error": err, "offsets": offsets,
            "view": ov.astype(np.int32), "xy": xy.astype(np.int64), "point2d": point2d.astype(np.int32),
            "view_offsets": view_offsets, "view_track": owner[order].astype(np.int32), "view_xy": xy[order].astype(np.int64)}


# ------------------------------------------------------------------------------------------------------------ COLMAP files
def write_model(folder, cameras, images, points3d, binary=True):
    """COLMAP's layouts, one record at a time.  cameras: [(camera_id, model_id, width, height, params)]; images:
    [(image_id, qvec, tvec, camera_id, name, [(x, y, point3D_id)])]; points3d: [(id, xyz, rgb, error, [(image_id, idx)])].
    Model id 1 is PINHOLE."""
    os.makedirs(folder, exist_ok=True)
    if binary:
        with open(os.path.join(folder, "cameras.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(cameras)))
            for cid, model, w, h, params in cameras:
                f.write(struct.pack("<iiQQ", cid, model, w, h) + struct.pack(f"<{len(params)}d", *params))
        with open(os.path.join(folder, "images.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(images)))
            for iid, q, t, cid, name, p2d in images:
                f.write(struct.pack("<idddddddi", iid, *q, *t, cid) + name.encode() + b"\0" + struct.pack("<Q", len(p2d)))
                for x, y, pid in p2d:
                    f.write(struct.pack("<ddq", x, y, pid))
        with open(os.path.join(folder, "points3D.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(points3d)))
            for pid, xyz, rgb, err, track in points3d:
                f.write(struct.pack("<QdddBBBd", pid, *xyz, *rgb, err) + struct.pack("<Q", len(track)))
                for iid, idx in track:
                    f.write(struct.pack("<ii", iid, idx))
        return
    with open(os.path.join(folder, "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n"
                f"# Number of cameras: {len(cameras)}\n")
        for cid, model, w, h, params in cameras:
            assert model == 1
            f.write(" ".join([str(cid), "PINHOLE", str(w), str(h)] + [repr(float(p)) for p in params]) + "\n")
    n_obs = sum(len(im[5]) for im in images)
    with open(os.path.join(folder, "images.txt"), "w") as f:
        f.write("# Image list with two lines of data per image:\n"
                "#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n#   POINTS2D[] as (X, Y, POINT3D_ID)\n"
                f"# Number of images: {len(images)}, mean observations per image: {float(n_obs) / len(images)!r}\n")
        for iid, q, t, cid, name, p2d in images:
            f.write(" ".join([str(iid)] + [repr(float(v)) for v in (*q, *t)] + [str(cid), name]) + "\n")
            f.write(" ".join(f"{float(x)!r} {float(y)!r} {int(pid)}" for x, y, pid in p2d) + "\n")
    n_track = sum(len(p[4]) for p in points3d)
    with open(os.path.join(folder, "points3D.txt"), "w") as f:
        mean = float(n_track) / len(points3d) if points3d else 0.0
        f.write("# 3D point list with one line of data per point:\n"
                "#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n"
                f"# Number of points: {len(points3d)}, mean track length: {mean!r}\n")
        for pid, xyz, rgb, err, track in points3d:
            f.write(" ".join([str(pid)] + [repr(float(v)) for v in xyz] + [str(int(c)) for c in rgb] + [repr(float(err))]
                             + [f"{int(i)} {int(k)}" for i, k in track]) + "\n")


def read_model(folder, binary=True):
    """(cameras, images, points3d) in write_model's layout, from either format."""
    cameras, images, points3d = [], [], []
    if binary:
        with open(os.path.join(folder, "cameras.bin"), "rb") as f:
            for _ in range(struct.unpack("<Q", f.read(8))[0]):
                cid, model, w, h = struct.unpack("<iiQQ", f.read(24))
                assert model == 1
                cameras.append((cid, model, w, h, list(struct.unpack("<4d", f.read(32)))))
            assert f.read() == b""
        with open(os.path.join(folder, "images.bin"), "rb") as f:
            for _ in range(struct.unpack("<Q", f.read(8))[0]):
                rec = struct.unpack("<idddddddi", f.read(64))
                name = b""
                while (c := f.read(1)) != b"\0":
                    name += c
                n = struct.unpack("<Q", f.read(8))[0]
                p2d = [struct.unpack("<ddq", f.read(24)) for _ in range(n)]
                images.append((rec[0], list(rec[1:5]), list(rec[5:8]), rec[8], name.decode(), p2d))
            assert f.read() == b""
        with open(os.path.join(folder, "points3D.bin"), "rb") as f:
            for _ in range(struct.unpack("<Q", f.read(8))[0]):
                rec = struct.unpack("<QdddBBBd", f.read(43))
                n = struct.unpack("<Q", f.read(8))[0]
                track = [struct.unpack("<ii", f.read(8)) for _ in range(n)]
                points3d.append((rec[0], list(rec[1:4]), list(rec[4:7]), rec[7], track))
            assert f.read() == b""
        return cameras, images, points3d

    def data_lines(name):
        with open(os.path.join(folder, name)) as f:
            return [line.rstrip("\n") for line in f if not line.startswith("#")]

    for line in data_lines("cameras.txt"):
        w = line.split()
        assert w[1] == "PINHOLE"
        cameras.append((int(w[0]), 1, int(w[2]), int(w[3]), [float(v) for v in w[4:]]))
    lines = data_lines("images.txt")
    for head, pts in zip(lines[0::2], lines[1::2]):
        w = head.split()
        p = pts.split()
        p2d = [(float(p[i]), float(p[i + 1]), int(p[i + 2])) for i in range(0, len(p), 3)]
        images.append((int(w[0]), [float(v) for v in w[1:5]], [float(v) for v in w[5:8]], int(w[8]), w[9], p2d))
    for line in data_lines("points3D.txt"):
        w = line.split()
        track = [(int(w[i]), int(w[i + 1])) for i in range(8, len(w), 2)]
        points3d.append((int(w[0]), [float(v) for v in w[1:4]], [int(v) for v in w[4:7]], float(w[7]), track))
    return cameras, images, points3d


def qvec_to_rotmat(q):
    """COLMAP's rotation of qvec (w, x, y, z)."""
    w, x, y, z = q
    return np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x * x - 2 * y * y]])


def check_model(folder, binary, extrinsic, H, W):
    """The model's invariants: every track element resolves to a 2-D point whose point3D_id is that track, every 2-D point
    is in exactly one track, qvec's rotation equals extrinsic to 1e-6 and the image sizes match the cameras (the PNGs under
    ../../images when they exist).  Returns (cameras, images, points3d)."""
    cameras, images, points3d = read_model(folder, binary)
    by_id = {im[0]: im for im in images}
    seen = set()
    for pid, _, _, _, track in points3d:
        for iid, idx in track:
            assert by_id[iid][5][idx][2] == pid, (pid, iid, idx)
            assert (iid, idx) not in seen
            seen.add((iid, idx))
    assert len(seen) == sum(len(im[5]) for im in images)
    cams = {c[0]: c for c in cameras}
    root = os.path.dirname(os.path.dirname(folder))
    for iid, q, t, cid, name, _ in images:
        R = qvec_to_rotmat(q)
        E = np.asarray(extrinsic[iid - 1], np.float64)
        assert np.abs(R - E[:, :3]).max() < 1e-6 and np.array_equal(np.asarray(t), E[:, 3])
        assert cams[cid][2:4] == (W, H)
        png = os.path.join(root, "images", name)
        if os.path.exists(png):
            from PIL import Image
            assert Image.open(png).size == (W, H)
    return cameras, images, points3d
