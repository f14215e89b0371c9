"""Point cloud and GLB export: the numpy oracle against the unmodified reference's GLB export and viewer (CPU), the .glb
writer (CPU), and the libovg point-cloud kernels / OmniVGGT.point_cloud against the oracle (GPU)."""
import os

import numpy as np
import pytest
import torch
from safetensors.torch import load_file

from conftest import GOLDEN
from oracle import pointcloud_oracle as PC
from oracle.make_golden_cloud import GLB_CASES, VIEWER_CASES, make_cloud_inputs
from ovg_support import dry, parse_glb, scene, sha256  # noqa: F401  (fixture)


def _gold():
    """The golden with its inputs: the reference's depth points and cameras are stored, the other inputs are regenerated
    by make_cloud_inputs and must match the stored digests."""
    g = {k: v.numpy() for k, v in load_file(os.path.join(GOLDEN, "point_cloud.safetensors")).items()}
    inp = make_cloud_inputs()
    for k in ("images", "depth_conf", "world_points", "world_points_conf"):
        g[k] = inp[k][0].numpy()
        assert sha256(g[k], hex=False) == g[f"{k}_sha256"].tobytes(), f"make_cloud_inputs no longer reproduces {k}"
    return g


def _source(g, src):
    return (g["world_points_from_depth"], g["depth_conf"]) if src == "depth" else (g["world_points"], g["world_points_conf"])


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_inputs_cover_the_edge_cases():
    g = _gold()
    cols = PC.colors_u8(g["images"])
    s = cols.astype(int).sum(1)
    assert (s == 15).any() and (s == 16).any() and (cols == 240).any() and (cols == 241).any()
    assert ((cols > 240).all(1)).any() and (s == 0).any()
    assert (np.unique(g["depth_conf"], return_counts=True)[1] > 1000).any()
    assert (g["world_points"] < 0).any() and (g["world_points"] == 0).any()


@pytest.mark.parametrize("i", range(len(GLB_CASES)))
def test_oracle_matches_reference_glb_export(i):
    g = _gold()
    src, pct, frame, black, white = GLB_CASES[i]
    world, conf = _source(g, src)
    o = PC.point_cloud(world, conf, g["images"], g["extrinsic"], pct, 1e-5, frame, black, white)
    if len(o["points"]) == 0:                                    # the reference's placeholder (visual_util.py:226-229)
        assert int(g[f"glb{i}_count"]) == 1 and o["scale"] == 1.0
        assert sha256(np.array([[1, 0, 0]]), hex=False) == g[f"glb{i}_points_sha256"].tobytes()
        assert sha256(np.array([[255, 255, 255]]), hex=False) == g[f"glb{i}_colors_sha256"].tobytes()
    else:
        assert len(o["points"]) == int(g[f"glb{i}_count"]) and o["points"].dtype == np.float32
        assert sha256(o["points"], hex=False) == g[f"glb{i}_points_sha256"].tobytes()
        assert sha256(o["colors"], hex=False) == g[f"glb{i}_colors_sha256"].tobytes()
        assert set(np.unique(o["frame"])) <= ({0, 1, 2} if frame is None else {frame})
        assert (np.diff(o["frame"]) >= 0).all()
    assert float(o["scale"] * 0.05) == float(g[f"glb{i}_radius"])          # cam_width = scene_scale * 0.05, fp32
    assert float(o["conf_threshold"]) == float(g[f"glb{i}_thr"])
    assert np.abs(o["align"] - g[f"glb{i}_align"]).max() <= 1e-6


@pytest.mark.parametrize("i", range(len(VIEWER_CASES)))
def test_oracle_matches_reference_viewer(i):
    """The viewer's initial cloud is the depth cloud with floor 0.1, recentred on the mean of all points."""
    g = _gold()
    pct, black, white = VIEWER_CASES[i]
    o = PC.point_cloud(g["world_points_from_depth"], g["depth_conf"], g["images"], g["extrinsic"], pct, 0.1, None, black, white)
    assert len(o["points"]) == int(g[f"viewer{i}_count"])
    assert sha256(o["points"] - o["center"], hex=False) == g[f"viewer{i}_points_sha256"].tobytes()
    assert sha256(o["colors"], hex=False) == g[f"viewer{i}_colors_sha256"].tobytes()


def _read_cloud(doc, binary):
    prim = doc["meshes"][0]["primitives"][0]
    assert prim["mode"] == 0
    acc = doc["accessors"]
    pos, col = acc[prim["attributes"]["POSITION"]], acc[prim["attributes"]["COLOR_0"]]
    assert pos["componentType"] == 5126 and pos["type"] == "VEC3"
    assert col["componentType"] == 5121 and col["type"] == "VEC4" and col["normalized"] is True
    views = doc["bufferViews"]
    for a in (pos, col):
        assert views[a["bufferView"]]["byteOffset"] % 4 == 0
    assert doc["buffers"][0]["byteLength"] <= len(binary)
    vp, vc = views[pos["bufferView"]], views[col["bufferView"]]
    p = np.frombuffer(binary, np.float32, pos["count"] * 3, vp["byteOffset"]).reshape(-1, 3)
    c = np.frombuffer(binary, np.uint8, col["count"] * 4, vc["byteOffset"]).reshape(-1, 4)
    assert pos["count"] == col["count"]
    assert pos["min"] == [float(v) for v in p.min(0)] and pos["max"] == [float(v) for v in p.max(0)]
    return p, c


def test_write_glb_round_trip(tmp_path):
    from omnivggt_official_b200.glb import write_glb
    g = _gold()
    o = PC.point_cloud(g["world_points_from_depth"], g["depth_conf"], g["images"], g["extrinsic"], 50.0, 1e-5, None, True, True)
    for n in (len(o["points"]), 1, 2, 3):                      # 2 and 3 points: chunk padding
        cloud = {"points": torch.from_numpy(o["points"][:n]), "colors": torch.from_numpy(o["colors"][:n]), "align": o["align"]}
        path = tmp_path / "scene.glb"
        write_glb(str(path), cloud)
        doc, binary = parse_glb(path.read_bytes())
        assert doc["asset"]["version"] == "2.0"
        p, c = _read_cloud(doc, binary)
        assert np.array_equal(p, o["points"][:n]) and np.array_equal(c[:, :3], o["colors"][:n]) and (c[:, 3] == 255).all()
        m = np.array(doc["nodes"][0]["matrix"]).reshape(4, 4).T            # column-major
        assert np.array_equal(m, o["align"])


def test_write_glb_empty_cloud_is_the_reference_placeholder(tmp_path):
    from omnivggt_official_b200.glb import write_glb
    path = tmp_path / "empty.glb"
    write_glb(str(path), {"points": np.zeros((0, 3), np.float32), "colors": np.zeros((0, 3), np.uint8), "align": np.eye(4)})
    doc, binary = parse_glb(path.read_bytes())
    p, c = _read_cloud(doc, binary)
    assert np.array_equal(p, [[1, 0, 0]]) and np.array_equal(c, [[255, 255, 255, 255]])


def test_dry_run_call_order_and_one_host_read(dry):
    """conf mask -> count -> centre -> one host read of the kept count and the first camera; the same calls for 1 and 24
    views.  The recorder's kept count is 0, so the cloud ends there."""
    from omnivggt_official_b200 import OmniVGGT
    seqs = []
    for S in (1, 24):
        dry.calls.clear()
        out = OmniVGGT.point_cloud(scene(S, 6, 8, distinct_cameras=True), mask_white_bg=True)
        names = dry.names()
        assert names == ["ovg_conf_percentile_mask", "ovg_point_cloud_workspace_bytes", "ovg_point_cloud_count",
                         "ovg_point_cloud_center", "host_read"]
        assert dry.calls[2][1][2:7] == (S, 6, 8, 0, 1)
        assert out["points"].shape == (0, 3) and torch.equal(out["align"], OmniVGGT._align(torch.eye(4)[:3].double()))
        seqs.append(names)
    assert seqs[0] == seqs[1] and len(dry.reads) == 2
    dry.calls.clear()
    pred = scene(5, 6, 8, distinct_cameras=True)
    out = OmniVGGT.point_cloud(pred, frame=3)
    assert dry.calls[2][1][2] == 1                                       # one view after the frame selection
    assert torch.equal(out["align"], OmniVGGT._align(pred["extrinsic"][0, 3].double()))
    assert len(dry.reads) == 3


def test_errors_before_any_device_work(dry):
    from omnivggt_official_b200 import OmniVGGT
    pred = scene(4, 6, 8, distinct_cameras=True)
    with pytest.raises(ValueError, match="source"):
        OmniVGGT.point_cloud(pred, source="normals")
    for pct in (-1.0, 100.5):
        with pytest.raises(ValueError, match="conf_percent"):
            OmniVGGT.point_cloud(pred, conf_percent=pct)
    with pytest.raises(ValueError, match="conf_floor"):
        OmniVGGT.point_cloud(pred, conf_floor=-1.0)
    for f in (4, -1):
        for mask_sky in (False, True):
            with pytest.raises(IndexError):
                OmniVGGT.point_cloud(pred, frame=f, mask_sky=mask_sky)
    with pytest.raises(ValueError, match="mask_sky"):
        OmniVGGT.point_cloud(pred, mask_sky=torch.zeros(4, 8, 6, dtype=torch.bool))
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
def _device_cloud(world, conf, images, extrinsic, **kw):
    from omnivggt_official_b200 import OmniVGGT
    pred = {"images": torch.from_numpy(images).cuda(), "extrinsic": torch.from_numpy(extrinsic).cuda(),
            "world_points_from_depth": torch.from_numpy(world).cuda(), "depth_conf": torch.from_numpy(conf).cuda()}
    out = OmniVGGT.point_cloud(pred, **kw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _check_against_oracle(d, world, conf, images, extrinsic, pct, floor, frame, black, white):
    """numpy's threshold to the bit, and bit-equal points / colours / frames."""
    od = PC.point_cloud(world, conf, images, extrinsic, pct, floor, frame, black, white)
    assert float(d["conf_threshold"]) == float(od["conf_threshold"]), (d["conf_threshold"], od["conf_threshold"])
    assert np.array_equal(d["points"], od["points"]) and np.array_equal(d["colors"], od["colors"])
    assert np.array_equal(d["frame"], od["frame"]) and d["frame"].dtype == np.int32
    pts = world if frame is None else world[frame]
    assert np.abs(d["center"] - od["center"]).max() <= 2e-6 * np.abs(pts).max()
    assert abs(float(d["scale"]) - float(od["scale"])) <= 1e-5 * float(od["scale"])
    assert np.abs(d["align"] - od["align"]).max() <= 1e-6
    return od


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(GLB_CASES)))
def test_point_cloud_kernels_match_golden(i):
    g = _gold()
    src, pct, frame, black, white = GLB_CASES[i]
    world, conf = _source(g, src)
    d = _device_cloud(world, conf, g["images"], g["extrinsic"], conf_percent=pct, frame=frame, mask_black_bg=black,
                      mask_white_bg=white)
    _check_against_oracle(d, world, conf, g["images"], g["extrinsic"], pct, 1e-5, frame, black, white)
    if len(d["points"]) == 0:
        assert float(d["scale"]) == 1.0 and d["colors"].shape == (0, 3)
    else:
        assert float(d["conf_threshold"]) == float(g[f"glb{i}_thr"])
        assert len(d["points"]) == int(g[f"glb{i}_count"])
        assert sha256(d["points"], hex=False) == g[f"glb{i}_points_sha256"].tobytes()
        assert sha256(d["colors"], hex=False) == g[f"glb{i}_colors_sha256"].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(VIEWER_CASES)))
def test_point_cloud_reproduces_viewer(i):
    g = _gold()
    pct, black, white = VIEWER_CASES[i]
    d = _device_cloud(g["world_points_from_depth"], g["depth_conf"], g["images"], g["extrinsic"], conf_percent=pct,
                      conf_floor=0.1, mask_black_bg=black, mask_white_bg=white)
    _check_against_oracle(d, g["world_points_from_depth"], g["depth_conf"], g["images"], g["extrinsic"], pct, 0.1, None,
                          black, white)
    if len(d["points"]) == int(g[f"viewer{i}_count"]):       # recentring: the centre is checked against the oracle above
        assert sha256(d["colors"], hex=False) == g[f"viewer{i}_colors_sha256"].tobytes()


def _large_inputs(S=24, H=518, W=518, seed=7):
    g = torch.Generator().manual_seed(seed)
    world = torch.randn(S, H, W, 3, generator=g) * 3.0
    world[:, ::5] = 0.0
    world[..., 1::3, 2] = world[0, 0, 1, 2]
    conf = 1.0 + torch.rand(S, H, W, generator=g).pow(3) * 8.0
    conf[..., ::4] = conf[0, 0, 0]
    conf[3] = 0.0
    images = torch.rand(S, 3, H, W, generator=g)
    images[:, :, :40] = 0.0
    images[:, :, 40:80] = 1.0
    ext = torch.eye(4)[:3].repeat(S, 1, 1) + 0.1 * torch.randn(S, 3, 4, generator=g)
    return world.numpy(), conf.numpy(), images.numpy(), ext.numpy()


@pytest.mark.gpu
def test_point_cloud_large_scene_matches_numpy_and_is_deterministic():
    """24 views @ 518^2 (6.4 M points) with negatives, zeros and heavy ties; two runs are bit-identical."""
    world, conf, images, ext = _large_inputs()
    kw = dict(conf_percent=30.0, mask_black_bg=True, mask_white_bg=True)
    d = _device_cloud(world, conf, images, ext, **kw)
    _check_against_oracle(d, world, conf, images, ext, 30.0, 1e-5, None, True, True)
    d2 = _device_cloud(world, conf, images, ext, **kw)
    for k in d:
        assert np.array_equal(d[k], d2[k]), k


@pytest.mark.gpu
def test_model_point_cloud_api():
    """model.point_cloud(model.postprocess(model(...))) agrees with the oracle on the same predictions, and gives the same
    cloud when postprocess() has not run (the depth points are then unprojected inside)."""
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
    raw = m(depth_gt_index=[1], camera_gt_index=[0], **inp)
    direct = m.point_cloud(dict(raw), conf_percent=25.0, mask_black_bg=True)
    pred = m.postprocess(raw)
    cloud = m.point_cloud(pred, conf_percent=25.0, mask_black_bg=True)
    torch.cuda.synchronize()
    d = {k: v.cpu().numpy() for k, v in cloud.items()}
    world = pred["world_points_from_depth"][0].cpu().numpy()
    conf = pred["depth_conf"][0].cpu().numpy()
    images = pred["images"][0].float().cpu().numpy()
    ext = pred["extrinsic"][0].cpu().numpy()
    _check_against_oracle(d, world, conf, images, ext, 25.0, 1e-5, None, True, False)
    for k in cloud:
        assert torch.equal(cloud[k], direct[k]), k
    pm = m.point_cloud(pred, source="pointmap", frame=2, conf_percent=10.0)
    dp = {k: v.cpu().numpy() for k, v in pm.items()}
    _check_against_oracle(dp, pred["world_points"][0].cpu().numpy(), pred["world_points_conf"][0].cpu().numpy(), images, ext,
                          10.0, 1e-5, 2, False, False)
    assert (dp["frame"] == 2).all()
