"""Triangle mesh of the point maps (reference omnivggt/viz.py:40-89 pts3d_to_trimesh + cat_meshes) and its GLB export.
CPU: the numpy oracle against the UNMODIFIED reference's outputs (tests/golden/mesh.safetensors), the GLB layout against the
reference layout, the .glb writer, a dry run of the library calls, and the errors.
GPU: libovg's ovg_mesh_* / OmniVGGT.mesh / the geometry drop-ins against the oracle bit for bit, 24 views of 518^2, single
views, repeats, and the mini model."""
import os

import numpy as np
import pytest
import torch
from safetensors.torch import load_file

from conftest import GOLDEN
from oracle import mesh_oracle as MO
from oracle.make_golden_cloud import GLB_CASES
from oracle.make_golden_mesh import cloud_inputs, glb_case_views, make_cases
from ovg_support import dry, parse_glb, scene, sha256  # noqa: F401  (fixture)

GOLD = {k: v.numpy() for k, v in load_file(os.path.join(GOLDEN, "mesh.safetensors")).items()}
CASES = make_cases()
NAMES = sorted(CASES)
KEYS = ("vertices", "face_colors", "faces")


def _check_golden(key, m):
    assert len(m["faces"]) == int(GOLD[f"{key}_count"])
    for k in KEYS:
        assert sha256(m[k], hex=False) == GOLD[f"{key}_{k}_sha256"].tobytes(), (key, k)


def _np(d):
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in d.items()}


def _source(g, src):
    return (g["world_points_from_depth"], g["depth_conf"]) if src == "depth" else (g["world_points"], g["world_points_conf"])


def _pred(g, device="cuda"):
    keys = ("images", "extrinsic", "world_points_from_depth", "depth_conf", "world_points", "world_points_conf")
    return {k: torch.from_numpy(np.ascontiguousarray(g[k]))[None].to(device) for k in keys}


def _expanded_forward(ref_views, glb):
    """(the vertices of the reference layout's (tl, tr, bl) and (tr, bl, br) faces, view by view; the GLB layout's
    positions[indices])."""
    fwd = []
    for cols, pts, keep in ref_views:
        m = MO.pts3d_to_trimesh(cols, pts, keep)
        c1, c3 = MO.class_counts(keep)
        f = np.concatenate((m["faces"][:c1], m["faces"][2 * c1:2 * c1 + c3]))
        fwd.append(m["vertices"][f])
    return np.concatenate(fwd).reshape(-1, 3, 3), glb["positions"][glb["indices"]]


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("i", range(len(GLB_CASES)))
def test_oracle_matches_reference_golden(i):
    g = cloud_inputs()
    src, pct, frame, black, white = GLB_CASES[i]
    world, conf = _source(g, src)
    o = MO.mesh(world, conf, g["images"], g["extrinsic"], pct, 1e-5, frame, black, white)
    _check_golden(f"glb{i}", o)
    assert o["faces"].dtype == np.int64 and o["face_colors"].dtype == np.uint8 and o["vertices"].dtype == np.float32


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_golden_cases(name):
    _check_golden(name, MO.cat_meshes([MO.pts3d_to_trimesh(*v) for v in CASES[name]]))


@pytest.mark.parametrize("i", range(len(GLB_CASES)))
def test_glb_layout_expands_to_the_forward_faces(i):
    g = cloud_inputs()
    src, pct, frame, black, white = GLB_CASES[i]
    world, conf = _source(g, src)
    glb = MO.mesh(world, conf, g["images"], g["extrinsic"], pct, 1e-5, frame, black, white, layout="glb")
    ref, got = _expanded_forward(glb_case_views(g, GLB_CASES[i]), glb)
    assert np.array_equal(ref, got) and glb["indices"].dtype == np.int32
    used = glb["indices"].reshape(-1)
    assert len(np.unique(used)) == len(glb["positions"])                # every vertex is used
    n_ref = int(GOLD[f"glb{i}_count"])
    assert 2 * len(glb["indices"]) == n_ref


def _read_mesh(doc, binary):
    prim = doc["meshes"][0]["primitives"][0]
    assert prim["mode"] == 4
    assert doc["materials"][prim["material"]]["doubleSided"] is True
    acc, views = doc["accessors"], doc["bufferViews"]
    pos, col, ind = acc[prim["attributes"]["POSITION"]], acc[prim["attributes"]["COLOR_0"]], acc[prim["indices"]]
    assert pos["componentType"] == 5126 and pos["type"] == "VEC3"
    assert col["componentType"] == 5121 and col["type"] == "VEC4" and col["normalized"] is True
    assert ind["componentType"] == 5125 and ind["type"] == "SCALAR"
    assert views[pos["bufferView"]]["target"] == 34962 and views[col["bufferView"]]["target"] == 34962
    assert views[ind["bufferView"]]["target"] == 34963
    for a in (pos, col, ind):
        v = views[a["bufferView"]]
        assert v["byteOffset"] % 4 == 0 and v["byteOffset"] + v["byteLength"] <= doc["buffers"][0]["byteLength"] <= len(binary)
    p = np.frombuffer(binary, np.float32, pos["count"] * 3, views[pos["bufferView"]]["byteOffset"]).reshape(-1, 3)
    c = np.frombuffer(binary, np.uint8, col["count"] * 4, views[col["bufferView"]]["byteOffset"]).reshape(-1, 4)
    i = np.frombuffer(binary, np.uint32, ind["count"], views[ind["bufferView"]]["byteOffset"]).reshape(-1, 3)
    assert pos["count"] == col["count"] and ind["count"] % 3 == 0
    assert pos["min"] == [float(v) for v in p.min(0)] and pos["max"] == [float(v) for v in p.max(0)]
    return p, c, i


def test_write_mesh_glb_parses(tmp_path):
    from omnivggt_official_b200.glb import write_mesh_glb
    g = cloud_inputs()
    o = MO.mesh(g["world_points_from_depth"], g["depth_conf"], g["images"], g["extrinsic"], 50.0, layout="glb")
    for k in (len(o["indices"]), 1, 2, 3):                      # few faces: chunk padding
        idx = o["indices"][:k]
        used = np.unique(idx)
        mesh = {"positions": torch.from_numpy(o["positions"][used]), "colors": torch.from_numpy(o["colors"][used]),
                "indices": torch.from_numpy(np.searchsorted(used, idx).astype(np.int32)), "align": o["align"]}
        path = tmp_path / "mesh.glb"
        write_mesh_glb(str(path), mesh)
        doc, binary = parse_glb(path.read_bytes())
        assert doc["asset"]["version"] == "2.0" and doc["scenes"][doc["scene"]]["nodes"] == [0]
        p, c, i = _read_mesh(doc, binary)
        assert np.array_equal(p[i], o["positions"][idx]) and np.array_equal(c[:, :3], o["colors"][used])
        assert (c[:, 3] == 255).all()
        m = np.array(doc["nodes"][0]["matrix"]).reshape(4, 4).T            # column-major
        assert np.array_equal(m, o["align"])


def test_write_mesh_glb_empty_and_non_finite(tmp_path):
    from omnivggt_official_b200.glb import mesh_glb_bytes, write_mesh_glb
    path = tmp_path / "empty.glb"
    write_mesh_glb(str(path), {"positions": np.zeros((0, 3), np.float32), "colors": np.zeros((0, 3), np.uint8),
                               "indices": np.zeros((0, 3), np.int32), "align": np.eye(4)})
    doc, binary = parse_glb(path.read_bytes())
    assert binary == b"" and doc["scenes"] == [{}] and doc["scene"] == 0 and "meshes" not in doc
    pos = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    mesh = {"positions": pos, "colors": np.zeros((3, 3), np.uint8), "indices": np.array([[0, 1, 2]], np.int32)}
    _read_mesh(*parse_glb(mesh_glb_bytes(mesh)))
    for bad in (np.nan, np.inf, -np.inf):
        pos[1, 2] = bad
        with pytest.raises(ValueError, match="finite"):
            mesh_glb_bytes(mesh)
    pos[1, 2] = 0.0
    with pytest.raises(ValueError, match="indices"):
        mesh_glb_bytes({**mesh, "indices": np.array([[0, 1, 3]], np.int32)})


@pytest.mark.parametrize("layout", ["reference", "glb"])
def test_dry_run_call_order_and_launches(dry, layout):
    """conf mask -> ovg_mesh_count -> one host read -> faces / compact; the same calls for 1 and 24 views."""
    from omnivggt_official_b200 import OmniVGGT
    last = "ovg_mesh_faces" if layout == "reference" else "ovg_mesh_compact"
    seqs = []
    for S in (1, 24):
        dry.calls.clear()
        out = OmniVGGT.mesh(scene(S, 6, 8), layout=layout, mask_white_bg=True)
        names = dry.names()
        assert names == ["ovg_conf_percentile_mask", "ovg_mesh_workspace_bytes", "ovg_mesh_count", "host_read", last]
        _, cnt = dry.calls[2]
        assert cnt[2:7] == (S, 6, 8, 0, 1)
        seqs.append(names)
        assert "align" in out and "conf_threshold" in out
    assert seqs[0] == seqs[1] and len(dry.reads) == 2
    dry.calls.clear()
    OmniVGGT.mesh(scene(5, 6, 8), frame=3)
    assert dry.calls[2][1][2] == 1                                       # one view after the frame selection


def test_errors_before_any_device_work(dry):
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.geometry import cat_meshes, pts3d_to_trimesh
    pred = scene(4, 6, 8)
    with pytest.raises(ValueError, match="source"):
        OmniVGGT.mesh(pred, source="normals")
    for pct in (-1.0, 100.5):
        with pytest.raises(ValueError, match="conf_percent"):
            OmniVGGT.mesh(pred, conf_percent=pct)
    with pytest.raises(ValueError, match="conf_floor"):
        OmniVGGT.mesh(pred, conf_floor=-1.0)
    with pytest.raises(ValueError, match="layout"):
        OmniVGGT.mesh(pred, layout="trimesh")
    for f in (4, -1):
        with pytest.raises(IndexError):
            OmniVGGT.mesh(pred, frame=f)
    with pytest.raises(ValueError, match="img"):
        pts3d_to_trimesh(np.zeros((4, 5, 4)), np.zeros((4, 5, 4)))
    with pytest.raises(ValueError, match="pts3d"):
        pts3d_to_trimesh(np.zeros((4, 5, 3)), np.zeros((5, 4, 3)))
    with pytest.raises(ValueError, match="valid"):
        pts3d_to_trimesh(np.zeros((4, 5, 3)), np.zeros((4, 5, 3)), np.ones((5, 4), bool))
    with pytest.raises(ValueError):
        cat_meshes([])
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
def _check_device_against_oracle(d, world, conf, images, ext, pct, frame, black, white, layout):
    """numpy's threshold to the bit, and bit-equal to the oracle."""
    od = MO.mesh(world, conf, images, ext, pct, 1e-5, frame, black, white, layout=layout)
    assert float(d["conf_threshold"]) == float(od["conf_threshold"]), (d["conf_threshold"], od["conf_threshold"])
    keys = KEYS if layout == "reference" else ("positions", "colors", "indices")
    for k in keys:
        assert d[k].dtype == od[k].dtype and np.array_equal(d[k], od[k]), k
    assert np.abs(d["align"] - od["align"]).max() <= 1e-6
    return od


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["reference", "glb"])
@pytest.mark.parametrize("i", range(len(GLB_CASES)))
def test_device_mesh_matches_oracle_and_golden(i, layout):
    from omnivggt_official_b200 import OmniVGGT
    g = cloud_inputs()
    src, pct, frame, black, white = GLB_CASES[i]
    world, conf = _source(g, src)
    d = _np(OmniVGGT.mesh(_pred(g), source=src, conf_percent=pct, frame=frame, mask_black_bg=black, mask_white_bg=white,
                          layout=layout))
    _check_device_against_oracle(d, world, conf, g["images"], g["extrinsic"], pct, frame, black, white, layout)
    if layout == "reference":
        _check_golden(f"glb{i}", d)


def _surface_pred(S=24, H=518, W=518, seed=9):
    from oracle.make_golden_matches import surface_views
    g = torch.Generator().manual_seed(seed)
    conf = 1.0 + torch.rand(S, H, W, generator=g) * 4.0
    conf[..., ::7] = conf[0, 0, 0]
    images = torch.rand(S, 3, H, W, generator=g)
    images[:, :, :30] = 1.0
    return {"world_points_from_depth": torch.from_numpy(surface_views(S, H, W, seed)), "depth_conf": conf, "images": images,
            "extrinsic": torch.eye(4)[:3].repeat(S, 1, 1) + 0.05 * torch.randn(S, 3, 4, generator=g)}


@pytest.mark.gpu
def test_24_views_518_match_oracle_and_repeat_bit_identically():
    from omnivggt_official_b200 import OmniVGGT, _lib
    host = _surface_pred()
    pred = {k: v.cuda() for k, v in host.items()}
    h = {k: v.numpy() for k, v in host.items()}
    lib = _lib.load()
    for layout in ("reference", "glb"):
        kw = dict(conf_percent=50.0, mask_white_bg=True, layout=layout)
        n0 = lib.ovg_launch_count()
        d = _np(OmniVGGT.mesh(pred, **kw))
        n1 = lib.ovg_launch_count()
        OmniVGGT.mesh(pred, frame=5, **kw)
        n2 = lib.ovg_launch_count()
        assert n1 - n0 == n2 - n1                                         # launches do not depend on the number of views
        _check_device_against_oracle(d, h["world_points_from_depth"], h["depth_conf"], h["images"], h["extrinsic"], 50.0,
                                     None, False, True, layout)
        again = _np(OmniVGGT.mesh(pred, **kw))
        for k in d:
            assert np.array_equal(d[k], again[k]), (layout, k)
    assert len(d["indices"]) > 100_000


@pytest.mark.gpu
def test_frame_equals_the_reference_on_that_view_alone():
    from omnivggt_official_b200 import OmniVGGT
    g = cloud_inputs()
    for f in range(3):
        d = _np(OmniVGGT.mesh(_pred(g), frame=f, conf_percent=40.0, mask_black_bg=True))
        keep, cols, _ = MO.keep_mask(g["depth_conf"][f][None], g["images"][f][None], 40.0, 1e-5, True, False,
                                     threshold=d["conf_threshold"])
        o = MO.pts3d_to_trimesh(cols[0], g["world_points_from_depth"][f], keep[0])
        for k in KEYS:
            assert np.array_equal(d[k], o[k]), (f, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_geometry_drop_ins_match_golden(name):
    from omnivggt_official_b200 import geometry
    views = CASES[name]
    ms = [geometry.pts3d_to_trimesh(img, pts, v) for img, pts, v in views]
    for m, (img, pts, v) in zip(ms, views):
        assert list(m) == list(KEYS) and m["faces"].is_cuda
        assert m["face_colors"].dtype == torch.from_numpy(img).dtype and m["faces"].dtype == torch.int64
        o = MO.pts3d_to_trimesh(img, pts, v)
        for k in KEYS:
            assert np.array_equal(m[k].cpu().numpy(), o[k]), k
    cat = geometry.cat_meshes(ms)
    assert list(cat) == list(KEYS)
    _check_golden(name, _np(cat))
    for m, (img, pts, v) in zip(ms, views):                           # inputs are not modified
        assert np.array_equal(m["faces"].cpu().numpy(), MO.pts3d_to_trimesh(img, pts, v)["faces"])
    # tensors already on the device, float32 colours of a uint8 case, and valid=None against all-true
    img, pts, v = views[0]
    a = geometry.pts3d_to_trimesh(torch.from_numpy(img.astype(np.float32)).cuda(), torch.from_numpy(pts).cuda(), v)
    assert a["face_colors"].dtype == torch.float32
    assert np.array_equal(a["face_colors"].cpu().numpy(), MO.pts3d_to_trimesh(img.astype(np.float32), pts, v)["face_colors"])
    b = geometry.pts3d_to_trimesh(img, pts, None)
    c = geometry.pts3d_to_trimesh(img, pts, np.ones(img.shape[:2], bool))
    assert torch.equal(b["faces"], c["faces"]) and torch.equal(b["face_colors"], c["face_colors"])


@pytest.mark.gpu
def test_model_mesh_api_and_glb_bytes():
    from test_model_gpu import model
    from omnivggt_official_b200.glb import mesh_glb_bytes
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
    raw = m(depth_gt_index=[1], camera_gt_index=[0], **inp)
    direct = m.mesh(dict(raw), conf_percent=25.0, mask_black_bg=True)
    pred = m.postprocess(raw)
    world = pred["world_points_from_depth"][0].cpu().numpy()
    conf = pred["depth_conf"][0].cpu().numpy()
    images = pred["images"][0].float().cpu().numpy()
    ext = pred["extrinsic"][0].cpu().numpy()
    ref = m.mesh(pred, conf_percent=25.0, mask_black_bg=True)
    for k in ref:
        assert torch.equal(ref[k], direct[k]), k
    _check_device_against_oracle(_np(ref), world, conf, images, ext, 25.0, None, True, False, "reference")
    glb = _np(m.mesh(pred, conf_percent=25.0, mask_black_bg=True, layout="glb"))
    od = _check_device_against_oracle(glb, world, conf, images, ext, 25.0, None, True, False, "glb")
    assert len(glb["indices"]) > 0
    assert mesh_glb_bytes(glb) == mesh_glb_bytes({**od, "align": glb["align"]})
    cloud = m.point_cloud(pred, conf_percent=25.0, mask_black_bg=True)
    assert torch.equal(cloud["align"].cpu(), torch.from_numpy(glb["align"]))
    pm = _np(m.mesh(pred, source="pointmap", frame=2, conf_percent=10.0))
    _check_device_against_oracle(pm, pred["world_points"][0].cpu().numpy(), pred["world_points_conf"][0].cpu().numpy(),
                                 images, ext, 10.0, 2, False, False, "reference")
