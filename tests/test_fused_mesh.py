"""Fused mesh (OmniVGGT.fused_mesh, csrc/tsdf.cuh): TSDF fusion of a scene's depth maps and one marching-cubes surface.
CPU: the C table against the oracle's rule and its properties over all 256 cases, the oracle's marching cubes on analytic
sphere and torus volumes, the oracle's fusion of exact depth maps of a sphere, the GLB round trip, and dry runs of the library
calls, host reads, argument errors and operand contracts.
GPU: the device against the oracle bit for bit (volume and mesh) on synthetic scenes, the mini model's forward and its
reconstruct, and 24 views of 518 x 518; the extract entry points alone on analytic volumes; run-to-run and poisoned-memory
identity; the GLB round trip of OmniVGGT.fused_mesh.

Which launch first writes each region of the fused-mesh workspace (read from csrc/):
  bounds       kept count and non-finite flag: cudaMemsetAsync in ovg_tsdf_bounds; coordinate columns: tsdf_fill_kernel;
               selection state and histograms: tsdf_select_init_kernel before each selection;
  bricks       marks: cudaMemsetAsync in ovg_tsdf_integrate, then tsdf_mark_kernel;
  counts       tile counts: tsdf_count_kernel (every brick); offsets and total: tile_scan_kernel; totals: tsdf_totals_kernel;
  edge indices tsdf_vertices_kernel, for every voxel of a brick chunk with an observed voxel (the only ones read)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import tsdf_oracle as TO
from ovg_support import install, parse_glb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "omnivggt-official_b200", "csrc")


# ------------------------------------------------------------------------------------------------------------------ scenes
def look_at(eye, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    """World-to-camera [R | t] (OpenCV: x right, y down, z forward) of a camera at eye looking at target."""
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, up)
    if np.linalg.norm(x) < 1e-6:
        x = np.cross(z, (1.0, 0.0, 0.0))
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return np.concatenate([R, -(R @ eye)[:, None]], 1)


def _hit_sphere(o, d, c, r):
    oc = o - c
    b = (d * oc).sum(-1)
    disc = b * b - ((oc * oc).sum(-1) - r * r)
    t = -b - np.sqrt(np.maximum(disc, 0))
    return np.where((disc > 0) & (t > 0), t, np.inf)


def _hit_box(o, d, lo, hi):
    with np.errstate(divide="ignore", invalid="ignore"):
        t0, t1 = (lo - o) / d, (hi - o) / d
    tn, tf = np.minimum(t0, t1).max(-1), np.maximum(t0, t1).min(-1)
    return np.where((tn <= tf) & (tn > 0), tn, np.inf)


SHAPES = {"sphere": [("s", (0.0, 0.0, 0.0), 1.0)],
          "box": [("b", (-0.8, -0.5, -0.6), (0.7, 0.6, 0.5))],
          "two": [("s", (-0.6, 0.1, 0.0), 0.55), ("b", (0.2, -0.5, -0.4), (1.0, 0.4, 0.5))]}


def synthetic_scene(kind, S, H, W, seed=0, radius=3.0):
    """Predictions of S cameras on a ring around ``kind`` with its exact depth maps (fp32 [1, S, H, W, 1]), the points they
    unproject to, colours from the surface position, and a confidence of 0 where a ray misses (so those pixels are not kept)."""
    rng = np.random.default_rng(seed)
    ext, intr = np.zeros((S, 3, 4)), np.zeros((S, 3, 3))
    depth, pts, img, conf = (np.zeros((S, H, W)), np.zeros((S, H, W, 3)), np.zeros((S, 3, H, W)), np.zeros((S, H, W)))
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    for f in range(S):
        a = 2 * np.pi * f / S + rng.uniform(-0.2, 0.2)
        eye = radius * np.array([np.cos(a), rng.uniform(-0.6, 0.6), np.sin(a)])
        E = look_at(eye)
        fx = fy = 0.9 * max(H, W) * rng.uniform(0.9, 1.1)
        K = np.array([[fx, 0, W / 2], [0, fy, H / 2], [0, 0, 1]])
        dirs_c = np.stack([(xs - K[0, 2]) / fx, (ys - K[1, 2]) / fy, np.ones_like(xs)], -1)
        dirs_w = dirs_c @ E[:, :3]                       # R^T d, not normalised: the hit distance along it is the depth
        o = np.broadcast_to(eye, dirs_w.shape)
        hits = []
        for sh in SHAPES[kind]:
            if sh[0] == "s":
                n = np.linalg.norm(dirs_w, axis=-1, keepdims=True)
                hits.append(_hit_sphere(o, dirs_w / n, np.array(sh[1]), sh[2]) / n[..., 0])
            else:
                hits.append(_hit_box(o, dirs_w, np.array(sh[1]), np.array(sh[2])))
        z = np.min(hits, 0)
        seen = np.isfinite(z)
        depth[f] = np.where(seen, z, 0.0)
        p = eye + dirs_w * depth[f][..., None]
        pts[f] = np.where(seen[..., None], p, 0.0)
        img[f] = np.where(seen, (0.5 + 0.45 * np.tanh(p.transpose(2, 0, 1))), 1.0)
        conf[f] = np.where(seen, 1.0 + rng.random((H, W)), 0.0)
        ext[f], intr[f] = E, K
    t = lambda a: torch.from_numpy(a.astype(np.float32))[None]
    return {"images": t(img), "depth": t(depth)[..., None], "depth_conf": t(conf), "world_points_from_depth": t(pts),
            "extrinsic": t(ext), "intrinsic": t(intr)}


def oracle_of(pred, resolution=512, conf_percent=10.0, conf_floor=1e-5):
    """TO.fuse on the device's own keep mask, points and cameras (scene._kept_views, tested elsewhere)."""
    from omnivggt_official_b200 import scene as SC
    images, (ext, intr), points, mask, _, _ = SC._kept_views(pred, "depth", conf_percent, conf_floor, None, 0, False,
                                                            cameras="predictions")
    S, _, H, W = images.shape
    depth = SC._of_scene(pred["depth"], 3, 0).float().reshape(S, H, W)
    np_ = lambda t: t.cpu().numpy()
    return TO.fuse(np_(depth), np_(mask), np_(images), np_(ext), np_(intr), np_(points), resolution)


# ------------------------------------------------------------------------------------------------------------------ mesh checks
def mesh_checks(pos, idx):
    """(Euler characteristic, signed volume) of a closed, consistently oriented 2-manifold; asserts that it is one."""
    tri = np.asarray(idx, np.int64)
    assert len(tri) and (tri[:, 0] != tri[:, 1]).all() and (tri[:, 1] != tri[:, 2]).all() and (tri[:, 0] != tri[:, 2]).all()
    directed = np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]])
    d = set(map(tuple, directed.tolist()))
    assert len(d) == len(directed), "a directed edge is used twice: inconsistent orientation"
    assert all((b, a) in d for a, b in d), "an edge has one triangle: the mesh is not closed"
    assert len(np.unique(tri)) == len(pos), "every vertex is referenced"
    # every vertex's triangles form one fan (a disk): the link of a vertex is one cycle
    nxt = {}
    for a, b, c in tri.tolist():
        for v, p, q in ((a, b, c), (b, c, a), (c, a, b)):
            nxt.setdefault(v, {})[p] = q
    for v, ring in nxt.items():
        start, k, steps = next(iter(ring)), None, 0
        k = ring[start]
        while k != start:
            k, steps = ring[k], steps + 1
            assert steps <= len(ring)
        assert steps + 1 == len(ring), f"vertex {v} is not manifold"
    E = len(directed) // 2
    p = np.asarray(pos, np.float64)[tri]
    vol = np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0
    return len(pos) - E + len(tri), vol


def analytic(kind, n=(36, 34, 32), s=0.1):
    """(tsdf fp32 [nz, ny, nx], origin, s, signed distance function, analytic volume): a sphere or a torus whose signed distance
    is truncated to +-4 voxels (and divided by it), every voxel observed."""
    nx, ny, nz = n
    origin = np.array([-nx / 2 * s + 0.013, -ny / 2 * s - 0.021, -nz / 2 * s + 0.007], np.float32)
    z, y, x = np.meshgrid(*(origin[a] + np.arange(n[a]) * np.float32(s) for a in (2, 1, 0)), indexing="ij")
    if kind == "sphere":
        r = 1.1
        sd = lambda x, y, z: np.sqrt(x * x + y * y + z * z) - r
        vol = 4 / 3 * np.pi * r ** 3
    else:
        R, r = 1.0, 0.45
        sd = lambda x, y, z: np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z) - r
        vol = 2 * np.pi ** 2 * R * r * r
    tsdf = np.clip(sd(x, y, z) / (4 * s), -1, 1).astype(np.float32)
    return tsdf, origin, np.float32(s), sd, vol


# ------------------------------------------------------------------------------------------------------------------ CPU: table
def _c_table(tmp_path):
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include "mc_table.h"\nint main(void) { for (int c = 0; c < 256; ++c) {\n'
                   '  printf("%d", ovg_mc_tri_count[c]); for (int i = 0; i < OVG_MC_MAX_TRIS * 3; ++i) '
                   'printf(" %d", ovg_mc_tri_edges[c][i]); printf("\\n"); } return 0; }\n')
    exe = tmp_path / "t"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", CSRC, str(src), "-o", str(exe)], check=True)
    rows = [list(map(int, l.split())) for l in subprocess.run([str(exe)], capture_output=True, text=True,
                                                               check=True).stdout.splitlines()]
    return np.array([r[0] for r in rows]), np.array([r[1:] for r in rows])


def test_c_table_is_the_oracles_rule(tmp_path):
    count, edges = _c_table(tmp_path)
    mx, want_count, want_edges = TO.mc_table()
    assert np.array_equal(count, want_count) and np.array_equal(edges, want_edges)
    with open(os.path.join(CSRC, "mc_table.h")) as f:
        assert f.read() == TO.mc_table_header()


def test_table_properties_over_all_cases():
    _, count, table = TO.mc_table()
    corners = TO.CORNERS.astype(np.float64)
    mid = np.array([(corners[a] + corners[b]) / 2 for a, b in TO.EDGES])
    for case in range(256):
        neg = [(case >> c) & 1 for c in range(8)]
        crossing = {e for e, (a, b) in enumerate(TO.EDGES) if neg[a] != neg[b]}
        tris = table[case, :3 * count[case]].reshape(-1, 3).tolist()
        assert set(np.ravel(tris).tolist()) == crossing, case
        directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
        assert len(set(directed)) == len(directed), case
        boundary = {e for e in directed if (e[1], e[0]) not in directed}
        assert sorted(boundary) == sorted(TO.face_segments(case)), case          # exactly its face segments, each once
        interior = [e for e in directed if e not in boundary]
        assert all((b, a) in interior for a, b in interior), case
        if sum(neg) == 1:
            c = neg.index(1)
            for a, b, d in tris:
                normal = np.cross(mid[b] - mid[a], mid[d] - mid[a])
                assert np.dot(normal, (mid[a] + mid[b] + mid[d]) / 3 - corners[c]) > 0, case


# ------------------------------------------------------------------------------------------------------------------ CPU: oracle
@pytest.mark.parametrize("kind,euler", [("sphere", 2), ("torus", 0)])
def test_oracle_marching_cubes_on_analytic_volumes(kind, euler):
    tsdf, origin, s, sd, vol = analytic(kind)
    color = np.full(tsdf.shape + (4,), 255, np.uint8)
    pos, cols, idx = TO.extract(tsdf, color, origin, s)
    chi, v = mesh_checks(pos, idx)
    assert chi == euler
    assert v > 0 and abs(v / vol - 1) < 0.02, (v, vol)
    p = pos.astype(np.float64)
    assert np.abs(sd(p[:, 0], p[:, 1], p[:, 2])).max() < 0.5 * s


# Bounds set from the oracle's run on this scene (radius 1, resolution 256, voxel 0.0085): mean distance 0.0045 (about half a
# voxel), 99th percentile 0.0151 (under two voxels).
SPHERE_MEAN, SPHERE_P99 = 0.008, 0.02


def test_oracle_fusion_of_exact_depth_maps_of_a_sphere():
    from omnivggt_official_b200 import scene as SC
    pred = {k: v[0] for k, v in synthetic_scene("sphere", 10, 64, 80, seed=1).items()}
    images, depth, ext, intr = (pred[k].numpy() for k in ("images", "depth", "extrinsic", "intrinsic"))
    mask = (pred["depth_conf"].numpy() > 1e-5).astype(np.uint8)
    r = TO.fuse(depth[..., 0], mask, images, ext, intr, pred["world_points_from_depth"].numpy(), 256)
    dist = np.abs(np.linalg.norm(r["positions"].astype(np.float64), axis=1) - 1.0)
    print(f"sphere fusion: {len(dist)} vertices, voxel {r['voxel_size']:.4f}, mean {dist.mean():.4f}, "
          f"p99 {np.percentile(dist, 99):.4f}")
    assert dist.mean() < SPHERE_MEAN and np.percentile(dist, 99) < SPHERE_P99
    assert SC._fusion_grid(*(np.array(b, np.float64) for b in TO.bounds(pred["world_points_from_depth"].numpy(),
                                                                           mask)[1:3]), 256)[1] == r["voxel_size"]


def test_write_mesh_glb_of_the_oracle_result(tmp_path):
    from omnivggt_official_b200.glb import write_mesh_glb
    tsdf, origin, s, _, _ = analytic("sphere", n=(20, 20, 20))
    pos, cols, idx = TO.extract(tsdf, np.full(tsdf.shape + (4,), 200, np.uint8), origin, s)
    path = str(tmp_path / "m.glb")
    write_mesh_glb(path, {"positions": pos, "colors": cols, "indices": idx, "align": np.eye(4)})
    doc, binary = parse_glb(open(path, "rb").read())
    assert doc["accessors"][0]["count"] == len(pos) and len(binary) > 0


# ------------------------------------------------------------------------------------------------------------------ CPU: dry runs
def _reader(kept=100, extent=1.0, bad=0.0, totals=(6, 8)):
    def read(t):
        if t.numel() == 20:
            host = t.double().clone()
            host[:8] = torch.tensor([kept, 0, 0, 0, extent, extent, extent, bad], dtype=torch.float64)
            return host
        return torch.tensor(totals, dtype=torch.int64)
    return read


def _pred(S=3, H=8, W=12):
    return {k: v for k, v in synthetic_scene("sphere", S, H, W).items()}


def test_dry_run_call_order_and_two_host_reads(monkeypatch):
    from omnivggt_official_b200 import OmniVGGT
    dry = install(monkeypatch, read=_reader())
    out = OmniVGGT.fused_mesh(_pred(), resolution=16)
    names = [n for n in dry.names() if n.startswith("ovg_tsdf") or n == "host_read"]
    assert names == ["ovg_tsdf_workspace_bytes", "ovg_tsdf_bounds", "host_read", "ovg_tsdf_workspace_bytes",
                     "ovg_tsdf_integrate", "ovg_tsdf_count", "host_read", "ovg_tsdf_extract"]
    assert len(dry.reads) == 2
    # the grid of an extent of 1 at resolution 16: voxel 1.1 / 16, 17 voxels per axis
    assert dry.args("ovg_tsdf_workspace_bytes")[1][:3] == (17, 17, 17)
    args = dry.args("ovg_tsdf_integrate")[0]
    assert args[8:11] == (17, 17, 17) and args[14] == np.float32(1.1 / 16) and args[15] == np.float32(4 * np.float32(1.1 / 16))
    assert out["positions"].shape == (6, 3) and out["indices"].shape == (8, 3) and out["indices"].dtype == torch.int32
    assert set(out) == {"positions", "colors", "indices", "conf_threshold", "align", "origin", "voxel_size"}


@pytest.mark.parametrize("reader", [dict(kept=0), dict(extent=0.0), dict(totals=(0, 0))])
def test_dry_run_empty_scene_has_no_extract(monkeypatch, reader):
    from omnivggt_official_b200 import OmniVGGT
    dry = install(monkeypatch, read=_reader(**reader))
    out = OmniVGGT.fused_mesh(_pred(), resolution=16)
    assert dry.count("ovg_tsdf_extract") == 0 and len(dry.reads) == (2 if "totals" in reader else 1)
    assert dry.count("ovg_tsdf_integrate") == ("totals" in reader)
    assert all(out[k].shape == (0, 3) for k in ("positions", "colors", "indices"))
    assert out["align"].shape == (4, 4) and out["origin"].shape == (3,) and out["voxel_size"].shape == ()


def test_dry_run_non_finite_kept_point_raises_after_the_first_read(monkeypatch):
    from omnivggt_official_b200 import OmniVGGT
    dry = install(monkeypatch, read=_reader(bad=1.0))
    with pytest.raises(ValueError, match="must be finite"):
        OmniVGGT.fused_mesh(_pred(), resolution=16)
    assert len(dry.reads) == 1 and dry.count("ovg_tsdf_integrate") == 0


def _without(*keys):
    return lambda p: {k: v for k, v in p.items() if k not in keys}


BAD_ARGS = {
    "resolution_float": (dict(resolution=64.0), None),
    "resolution_bool": (dict(resolution=True), None),
    "resolution_low": (dict(resolution=15), None),
    "resolution_high": (dict(resolution=513), None),
    "no_depth": (dict(), "depth"),
    "no_cameras": (dict(), "cameras"),
    "conf_percent": (dict(conf_percent=101.0), None),
    "conf_floor": (dict(conf_floor=-1.0), None),
    "mask_sky": (dict(mask_sky=torch.zeros(2, 8, 12, dtype=torch.bool)), None),
    "too_many_pixels": (dict(), "huge"),
}


def _bad_pred(what):
    p = _pred()
    if what == "depth":
        p.pop("depth")
    elif what == "cameras":
        p.pop("extrinsic")
    elif what == "huge":
        p["images"] = torch.zeros(1, 1, 1, 1, 1).expand(1, 3, 3, 2 ** 16, 2 ** 14)   # 3 x 2^30 pixels, no memory
    return p


@pytest.mark.parametrize("name", sorted(BAD_ARGS))
def test_argument_errors_before_any_library_call(monkeypatch, name):
    from omnivggt_official_b200 import OmniVGGT
    kw, what = BAD_ARGS[name]
    dry = install(monkeypatch)
    with pytest.raises(ValueError):
        OmniVGGT.fused_mesh(_bad_pred(what), **kw)
    assert dry.calls == [] and dry.reads == []


def test_argument_errors_under_python_O():
    code = ("import sys, torch; sys.path[:0] = [%r, %r]\n"
            "import test_fused_mesh as T\n"
            "from omnivggt_official_b200 import _lib, ops, OmniVGGT\n"
            "calls = []\n"
            "_lib.lib = lambda: calls.append(1)\n"
            "ops._on_device = lambda t: True\n"
            "for name, (kw, what) in sorted(T.BAD_ARGS.items()):\n"
            "    try:\n"
            "        OmniVGGT.fused_mesh(T._bad_pred(what), **kw)\n"
            "    except ValueError:\n"
            "        continue\n"
            "    raise SystemExit(name)\n"
            "assert not calls\n" % (ROOT, os.path.dirname(os.path.abspath(__file__))))
    r = subprocess.run([sys.executable, "-O", "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout + r.stderr


# Operand contracts of the ops wrappers: each well-formed call, then each operand broken in turn.
def _z(*shape, dtype=torch.float32):
    return torch.zeros(*shape, dtype=dtype)


F, H, W, NZ, NY, NX = 2, 4, 6, 3, 5, 7
U8 = torch.uint8
WRAPPERS = {
    "tsdf_bounds": (lambda ops, a: ops.tsdf_bounds(**a), dict(points=_z(F, H, W, 3), mask=_z(F, H, W, dtype=U8))),
    "tsdf_integrate": (lambda ops, a: ops.tsdf_integrate(shape=(NZ, NY, NX), origin=(0, 0, 0), voxel=0.1, trunc=0.4, **a),
                       dict(depth=_z(F, H, W), mask=_z(F, H, W, dtype=U8), images=_z(F, 3, H, W), extrinsic=_z(F, 3, 4),
                            intrinsic=_z(F, 3, 3), ws=_z(256, dtype=U8))),
    "TsdfMesher": (lambda ops, a: ops.TsdfMesher(origin=(0, 0, 0), voxel=0.1, **a), dict(tsdf=_z(NZ, NY, NX), ws=_z(256, dtype=U8))),
    "TsdfMesher.extract": (lambda ops, a: ops.TsdfMesher(_z(NZ, NY, NX), (0, 0, 0), 0.1).extract(m=1, k=1, **a),
                           dict(color=_z(NZ, NY, NX, 4, dtype=U8))),
}


def _broken(name):
    _, base = WRAPPERS[name]
    for op, t in base.items():
        wrong = torch.float64 if t.dtype != torch.float64 else torch.float32
        yield op, "dtype", t.to(wrong), TypeError
        yield op, "device", t, TypeError
        yield op, "shape", torch.zeros(*(t.shape[:-1] + (t.shape[-1] + 1,)), dtype=t.dtype)[None], ValueError
        if t.dim() > 1:
            yield op, "layout", torch.zeros(*t.shape[:-1], 2 * t.shape[-1], dtype=t.dtype)[..., ::2], ValueError


@pytest.mark.parametrize("name", sorted(WRAPPERS))
def test_ops_operand_contracts(monkeypatch, name):
    from omnivggt_official_b200 import ops
    call, base = WRAPPERS[name]
    dry = install(monkeypatch)
    call(ops, dict(base))                                               # well formed
    for op, how, bad, exc in _broken(name):
        dry.calls.clear()
        if how == "device":
            monkeypatch.setattr(ops, "_on_device", lambda t, bad=bad: t is not bad)
        with pytest.raises(exc, match=op if op != "ws" else None):
            call(ops, dict(base, **{op: bad}))
        assert [n for n in dry.names() if not n.endswith("_workspace_bytes") and n != "ovg_tsdf_count"] == [], (op, how)
        monkeypatch.setattr(ops, "_on_device", lambda t: True)


# ------------------------------------------------------------------------------------------------------------------ GPU
def _cuda(pred):
    return {k: v.cuda() for k, v in pred.items()}


def _as_np(t):
    return t.cpu().numpy()


def assert_equal_to_oracle(res, tsdf, color, want):
    assert want is not None and tsdf is not None
    assert np.array_equal(_as_np(tsdf).view(np.int32), want["tsdf"].view(np.int32)), "tsdf volume"
    assert np.array_equal(_as_np(color), want["color"]), "colour volume"
    assert np.array_equal(_as_np(res["positions"]).view(np.int32), want["positions"].view(np.int32)), "positions"
    assert np.array_equal(_as_np(res["colors"]), want["colors"]), "colors"
    assert np.array_equal(_as_np(res["indices"]), want["indices"]), "indices"
    assert np.array_equal(_as_np(res["origin"]), want["origin"]) and float(res["voxel_size"]) == want["voxel_size"]


def _device(pred, resolution, conf_percent=10.0):
    from omnivggt_official_b200 import scene as SC
    return SC._fusion(pred, resolution, conf_percent, 1e-5, 0, False)


SCENES = [("sphere", 8, 64, 80, 16, 0), ("sphere", 6, 100, 72, 100, 1), ("box", 12, 96, 128, 100, 2),
          ("two", 9, 160, 120, 512, 3), ("box", 7, 80, 64, 512, 4), ("two", 10, 72, 96, 16, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,S,H,W,resolution,seed", SCENES)
def test_device_equals_oracle_on_synthetic_scenes(kind, S, H, W, resolution, seed):
    pred = _cuda(synthetic_scene(kind, S, H, W, seed=seed))
    res, tsdf, color = _device(pred, resolution)
    want = oracle_of(pred, resolution)
    assert_equal_to_oracle(res, tsdf, color, want)
    assert len(want["indices"]) > 0 and (resolution < 100 or want["marked"].mean() < 1.0)
    print(f"{kind} S={S} {H}x{W} res={resolution}: grid {tsdf.shape}, {want['marked'].mean():.3f} of the bricks marked, "
          f"{len(want['positions'])} vertices, {len(want['indices'])} triangles")


@pytest.mark.gpu
def test_grids_leave_partial_bricks_on_every_axis():
    shapes = []
    for kind, S, H, W, resolution, seed in SCENES:
        _, tsdf, _ = _device(_cuda(synthetic_scene(kind, S, H, W, seed=seed)), resolution)
        shapes.append(tuple(tsdf.shape))
    assert any(all(n % 8 for n in sh) for sh in shapes), shapes
    assert {max(sh) for sh in shapes} == {17, 101, 513}, shapes


@pytest.mark.gpu
def test_mini_model_forward_and_reconstruct():
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
    raw = m(depth_gt_index=[1], camera_gt_index=[0], **inp)
    for pred in (dict(raw), m.postprocess(dict(raw))):                 # cameras decoded inside, then the predictions' own
        res, tsdf, color = _device(pred, 64, 25.0)
        assert_equal_to_oracle(res, tsdf, color, oracle_of(pred, 64, 25.0))
    inp = {k: v.cuda() for k, v in make_inputs(1, 10, 56, 56, seed=63).items()}
    rec = m.reconstruct(**inp, chunk=6, overlap=2)
    res, tsdf, color = _device(rec, 100, 25.0)
    assert_equal_to_oracle(res, tsdf, color, oracle_of(rec, 100, 25.0))     # the untrained views carve each other: empty


@pytest.mark.gpu
def test_24_views_of_518():
    pred = _cuda(synthetic_scene("two", 24, 518, 518, seed=7))
    res, tsdf, color = _device(pred, 512)
    assert_equal_to_oracle(res, tsdf, color, oracle_of(pred, 512))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,euler", [("sphere", 2), ("torus", 0)])
def test_extract_entry_points_on_analytic_volumes(kind, euler):
    from omnivggt_official_b200 import ops
    tsdf, origin, s, sd, vol = analytic(kind)
    g = np.random.default_rng(0)
    color = g.integers(0, 256, tsdf.shape + (4,), dtype=np.uint8)
    mc = ops.TsdfMesher(torch.from_numpy(tsdf).cuda(), origin, s)
    m, k = mc.totals.tolist()
    pos, cols, idx = mc.extract(torch.from_numpy(color).cuda(), m, k)
    want = TO.extract(tsdf, color, origin, s)
    for got, w in zip((pos, cols, idx), want):
        assert np.array_equal(_as_np(got), w)
    chi, v = mesh_checks(_as_np(pos), _as_np(idx))
    assert chi == euler and v > 0 and abs(v / vol - 1) < 0.02


@pytest.mark.gpu
def test_repeatable_and_independent_of_memory():
    from test_poison_gpu import check_case
    pred = _cuda(synthetic_scene("two", 8, 64, 96, seed=11))
    first = _device(pred, 100)
    again = _device(pred, 100)
    for a, b in zip(first, again):
        a, b = (a, b) if isinstance(a, dict) else ({"t": a}, {"t": b})
        for k in a:
            if torch.is_tensor(a[k]):
                bits = lambda t: t.reshape(-1).view(torch.uint8) if t.is_floating_point() else t
                assert torch.equal(bits(a[k]), bits(b[k])), k

    def run(P):
        res, tsdf, color = _device(pred, 100)
        return {"mesh": res, "tsdf": tsdf.view(torch.int32), "color": color}
    check_case("fused_mesh", run, finite=("positions", "origin", "voxel_size"))


@pytest.mark.gpu
def test_model_fused_mesh_glb_round_trip(tmp_path):
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.glb import write_mesh_glb
    out = OmniVGGT.fused_mesh(_cuda(synthetic_scene("sphere", 8, 64, 64, seed=2)), resolution=64, conf_percent=10.0)
    path = str(tmp_path / "fused.glb")
    write_mesh_glb(path, out)
    doc, binary = parse_glb(open(path, "rb").read())
    assert doc["accessors"][0]["count"] == len(out["positions"]) > 0 and len(binary) > 0
