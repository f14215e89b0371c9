"""Multi-view tracks and the COLMAP export (OmniVGGT.tracks, colmap.write_colmap).
CPU: the numpy oracle against a brute-force restatement of the star rule on hand-made match graphs, the quaternion helper
against the reference's mat_to_quat (tests/golden/colmap.json), the writer's bytes on a hand-built model, a dry run of the
library calls, and the errors.
GPU: OmniVGGT.tracks against the oracle bit for bit, run-to-run and poisoned-memory identity, the pixel-centre convention,
and the written folders of the mini model's forward and of a reconstruct.

Which launch first writes each region of the track workspace (read from csrc/):
  claim map      cudaMemsetAsync (-1) in ovg_tracks_assign, then the write kernel of each anchor step;
  running totals cudaMemsetAsync (0) of slot 0 in ovg_tracks_assign; slot (a + 1) & 1 by block 0 of step a's write kernel;
  tile counts    the count kernel of each step (2 tiles), track_claimed_kernel in the gather (V tiles);
  tile offsets   tile_scan_kernel after each of those;
  observations   and track starts: the write kernels, at the offsets their scan gives (only entries below the totals are read);
  rank map       track_view_kernel, for the claimed nodes that track_point_kernel reads;
  counts_out     track_counts_kernel."""
import json
import os
import struct

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import matches_oracle as MO
from oracle import tracks_oracle as TO
from oracle.make_golden_matches import surface_views

INT_KEYS = ("offsets", "view", "xy", "point2d", "view_offsets", "view_track", "view_xy", "colors")


# ------------------------------------------------------------------------------------------------------------------ CPU
def brute_star(n_kept, edges, min_views):
    """The star rule, one node at a time.  edges: [(i, k_i, j, k_j)] in either orientation."""
    adj = {}
    for i, ki, j, kj in edges:
        adj.setdefault((i, ki), {})[j] = kj
        adj.setdefault((j, kj), {})[i] = ki
    claimed, tracks = {}, []
    for a in range(len(n_kept)):
        new = []
        for k in range(n_kept[a]):
            if (a, k) in claimed:
                continue
            members = [(a, k)] + [(j, kj) for j, kj in sorted(adj.get((a, k), {}).items()) if j > a and (j, kj) not in claimed]
            if len(members) >= min_views:
                new.append(members)
        for t in new:                       # no two anchors of one step share a node: claiming after the step is the same
            for node in t:
                assert node not in claimed
                claimed[node] = len(tracks)
            tracks.append(t)
    return tracks


def oracle_tracks(n_kept, edges, min_views):
    matches = {}
    for i, ki, j, kj in edges:
        if i > j:
            i, ki, j, kj = j, kj, i, ki
        a, b = matches.setdefault((i, j), ([], []))
        if (ki, kj) not in zip(a, b):        # a pair given twice (or reversed) is one pair
            a.append(ki)
            b.append(kj)
    matches = {p: (np.array(a, np.int64), np.array(b, np.int64)) for p, (a, b) in matches.items()}
    offsets, ov, ok = TO.star_tracks(n_kept, matches, min_views)
    return [list(zip(ov[s:e].tolist(), ok[s:e].tolist())) for s, e in zip(offsets[:-1], offsets[1:])]


GRAPHS = {
    # view 0 pixel 0 -> 1:0 and 2:0, but 1:0 -> 2:1 (not transitive); 1:1 -> 2:2 anchors later
    "star_not_chain": ([2, 3, 3], [(0, 0, 1, 0), (0, 0, 2, 0), (1, 0, 2, 1), (1, 1, 2, 2), (0, 1, 2, 2)]),
    "claimed_partner": ([2, 2, 2], [(0, 0, 1, 0), (1, 0, 2, 0), (1, 1, 2, 1), (0, 1, 2, 1)]),
    "reversed_and_duplicate_pairs": ([3, 3, 2], [(1, 0, 0, 2), (0, 2, 1, 0), (2, 1, 0, 0), (2, 0, 1, 2), (1, 2, 2, 0)]),
    "empty_view": ([2, 0, 3], [(0, 0, 2, 1), (0, 1, 2, 0)]),
    "no_edges": ([2, 1], []),
}


def _random_graph(seed):
    rng = np.random.default_rng(seed)
    V = int(rng.integers(2, 7))
    n = rng.integers(0, 12, V).tolist()
    edges = []
    for i in range(V):
        for j in range(V):
            if i != j and rng.random() < 0.4:
                m = int(min(n[i], n[j]) * rng.random())
                a, b = rng.permutation(n[i])[:m], rng.permutation(n[j])[:m]       # a one-to-one matching
                edges += [(i, int(x), j, int(y)) for x, y in zip(a, b)]
    # (i, j) and (j, i) both drawn: keep the first, as reciprocal matchings of one pair agree
    seen, out = set(), []
    for i, ki, j, kj in edges:
        key = (min(i, j), max(i, j))
        if key in seen and (key, i) not in seen:
            continue
        seen.add(key)
        seen.add((key, i))
        out.append((i, ki, j, kj))
    return n, out


@pytest.mark.parametrize("name", sorted(GRAPHS) + [f"random{s}" for s in range(12)])
def test_oracle_equals_brute_force_star_rule(name):
    n, edges = GRAPHS[name] if name in GRAPHS else _random_graph(int(name[6:]))
    for min_views in range(1, len(n) + 1):
        assert oracle_tracks(n, edges, min_views) == brute_star(n, edges, min_views), min_views


def test_hand_made_graphs_give_the_documented_tracks():
    n, e = GRAPHS["star_not_chain"]
    assert oracle_tracks(n, e, 2) == [[(0, 0), (1, 0), (2, 0)], [(0, 1), (2, 2)]]          # 1:0 is claimed, 1:1's partner too
    assert oracle_tracks(n, e, 3) == [[(0, 0), (1, 0), (2, 0)]]
    assert oracle_tracks(n, e, 1) == [[(0, 0), (1, 0), (2, 0)], [(0, 1), (2, 2)], [(1, 1)], [(1, 2)], [(2, 1)]]
    n, e = GRAPHS["empty_view"]
    assert oracle_tracks(n, e, 1) == [[(0, 0), (2, 1)], [(0, 1), (2, 0)], [(2, 2)]]


def test_quaternion_helper_matches_reference_mat_to_quat():
    from omnivggt_official_b200.colmap import rotmat_to_qvec
    g = json.load(open(os.path.join(GOLDEN, "colmap.json")))
    R = np.array(g["rotations"])
    want = np.array(g["mat_to_quat_xyzw"])[:, [3, 0, 1, 2]]
    got = rotmat_to_qvec(R)
    assert np.abs(got - want).max() <= 1e-15
    assert (got[:, 0] >= 0).all() and np.allclose([TO.qvec_to_rotmat(q) for q in got], R, atol=1e-12)


def _two_view_model():
    """Two views of 2 x 2 pixels: two tracks (0:(1,0) <-> 1:(0,1), and a one-view point at 1:(1,1))."""
    images = torch.tensor([[[[0.0, 0.5], [1.0, 0.25]]] * 3, [[[0.1, 0.2], [0.3, 0.4]]] * 3], dtype=torch.float32)[None]
    ext = torch.tensor([[[1.0, 0, 0, 0.25], [0, 1, 0, -0.5], [0, 0, 1, 2]], [[0, -1.0, 0, 1], [1, 0, 0, 0], [0, 0, 1, 3]]])
    intr = torch.tensor([[[2.0, 0, 1], [0, 3, 1], [0, 0, 1]], [[4.0, 0, 1], [0, 5, 1], [0, 0, 1]]])
    tracks = {"points": torch.tensor([[0.5, -1.25, 3.0], [1e-3, 2.0, 0.1]], dtype=torch.float64),
              "colors": torch.tensor([[127, 127, 127], [102, 102, 102]], dtype=torch.uint8),
              "error": torch.tensor([0.125, float("inf")], dtype=torch.float64),
              "offsets": torch.tensor([0, 2, 3]), "view": torch.tensor([0, 1, 1], dtype=torch.int32),
              "xy": torch.tensor([[1, 0], [0, 1], [1, 1]]), "point2d": torch.tensor([0, 0, 1], dtype=torch.int32),
              "view_offsets": torch.tensor([0, 1, 3]), "view_track": torch.tensor([0, 0, 1], dtype=torch.int32),
              "view_xy": torch.tensor([[1, 0], [0, 1], [1, 1]]), "extrinsic": ext, "intrinsic": intr}
    return {"images": images}, tracks


def _expected_binary():
    q0, q1 = (1.0, 0.0, 0.0, 0.0), (0.7071067811865477, 0.0, 0.0, 0.7071067811865475)    # correctly rounded fp64
    cams = struct.pack("<Q", 2) + struct.pack("<iiQQ4d", 1, 1, 2, 2, 2.0, 3.0, 1.5, 1.5) \
        + struct.pack("<iiQQ4d", 2, 1, 2, 2, 4.0, 5.0, 1.5, 1.5)
    ims = struct.pack("<Q", 2) + struct.pack("<idddddddi", 1, *q0, 0.25, -0.5, 2.0, 1) + b"a.png\0" + struct.pack("<Q", 1) \
        + struct.pack("<ddq", 1.5, 0.5, 1) + struct.pack("<idddddddi", 2, *q1, 1.0, 0.0, 3.0, 2) + b"b.png\0" \
        + struct.pack("<Q", 2) + struct.pack("<ddq", 0.5, 1.5, 1) + struct.pack("<ddq", 1.5, 1.5, 2)
    pts = struct.pack("<Q", 2) + struct.pack("<QdddBBBd", 1, 0.5, -1.25, 3.0, 127, 127, 127, 0.125) + struct.pack("<Q", 2) \
        + struct.pack("<ii", 1, 0) + struct.pack("<ii", 2, 0) \
        + struct.pack("<QdddBBBd", 2, 1e-3, 2.0, 0.1, 102, 102, 102, float("inf")) + struct.pack("<Q", 1) + struct.pack("<ii", 2, 1)
    return {"cameras.bin": cams, "images.bin": ims, "points3D.bin": pts}


EXPECTED_TEXT = {
    "cameras.txt": "# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n"
                   "# Number of cameras: 2\n1 PINHOLE 2 2 2.0 3.0 1.5 1.5\n2 PINHOLE 2 2 4.0 5.0 1.5 1.5\n",
    "images.txt": "# Image list with two lines of data per image:\n#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n"
                  "#   POINTS2D[] as (X, Y, POINT3D_ID)\n# Number of images: 2, mean observations per image: 1.5\n"
                  "1 1.0 0.0 0.0 0.0 0.25 -0.5 2.0 1 a.png\n1.5 0.5 1\n"
                  "2 0.7071067811865477 0.0 0.0 0.7071067811865475 1.0 0.0 3.0 2 b.png\n0.5 1.5 1 1.5 1.5 2\n",
    "points3D.txt": "# 3D point list with one line of data per point:\n"
                    "#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n"
                    "# Number of points: 2, mean track length: 1.5\n"
                    "1 0.5 -1.25 3.0 127 127 127 0.125 1 0 2 0\n2 0.001 2.0 0.1 102 102 102 inf 2 1\n",
}


def test_write_colmap_bytes(tmp_path):
    from omnivggt_official_b200.colmap import write_colmap
    pred, tracks = _two_view_model()
    sb = write_colmap(str(tmp_path / "b"), pred, tracks, image_names=["a.png", "b.png"], images=False)
    for name, want in _expected_binary().items():
        assert open(os.path.join(sb, name), "rb").read() == want, name
    st = write_colmap(str(tmp_path / "t"), pred, tracks, image_names=["a.png", "b.png"], binary=False)
    for name, want in EXPECTED_TEXT.items():
        assert open(os.path.join(st, name)).read() == want, name
    assert TO.read_model(sb, True) == TO.read_model(st, False)
    TO.check_model(st, False, tracks["extrinsic"].numpy(), 2, 2)             # the PNGs were written: sizes checked too
    from PIL import Image
    assert np.array_equal(np.asarray(Image.open(tmp_path / "t" / "images" / "b.png"))[..., 0], [[25, 51], [76, 102]])
    TO.write_model(str(tmp_path / "o"), *TO.read_model(sb, True), binary=True)      # the spec writer gives the same bytes
    for name, want in _expected_binary().items():
        assert open(tmp_path / "o" / name, "rb").read() == want, name
    TO.write_model(str(tmp_path / "ot"), *TO.read_model(sb, True), binary=False)
    for name, want in EXPECTED_TEXT.items():
        assert open(tmp_path / "ot" / name).read() == want, name


def test_write_colmap_errors(tmp_path):
    from omnivggt_official_b200.colmap import write_colmap
    pred, tracks = _two_view_model()
    for names in (["a.png"], ["a.png", "a.png"], ["a.png", "x/b.png"], ["a.png", ""]):
        with pytest.raises(ValueError):
            write_colmap(str(tmp_path), pred, tracks, image_names=names)
    with pytest.raises(ValueError, match="scene"):
        write_colmap(str(tmp_path), {"images": pred["images"][:, :1]}, tracks)
    assert not os.path.exists(tmp_path / "sparse")


@pytest.fixture()
def dry(monkeypatch):
    """The C library replaced by a recorder, on CPU tensors; host reads counted (they read zeros)."""
    from omnivggt_official_b200 import _lib, ops

    class Rec:
        def __init__(self):
            self.calls, self.reads = [], 0

        def __getattr__(self, name):
            def fn(*a):
                self.calls.append((name, a))
                return 0
            return fn

    rec = Rec()

    def read(t):
        rec.reads += 1
        return torch.zeros_like(t, device="cpu")

    monkeypatch.setattr(_lib, "lib", lambda: rec)
    monkeypatch.setattr(_lib, "stream", lambda: 0)
    monkeypatch.setattr(ops, "_on_device", lambda t: True)
    monkeypatch.setattr(ops, "host_read", read)
    return rec


def _scene(S, H, W, seed=5):
    from test_matches import _scene as matches_scene
    pred = matches_scene(S, H, W, seed)
    pred["intrinsic"] = torch.tensor([[W * 0.9, 0, W / 2], [0, W * 0.9, H / 2], [0, 0, 1]]).repeat(1, S, 1, 1)
    return pred


@pytest.mark.parametrize("pairs,P", [([(0, 1)], 1), ([(3, 1), (1, 3), (0, 2)], 2), (None, 15), ([], 0)])
def test_dry_run_reads_once(dry, pairs, P):
    """One index build, one query, one assignment, one read; launches of the assignment do not depend on P; the pairs are
    normalised, merged and sorted, and without pairs the matcher still gets one."""
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = 6, 8, 10
    out = OmniVGGT.tracks(_scene(S, H, W), pairs, min_views=1)
    assert [n for n, _ in dry.calls] == ["ovg_conf_percentile_mask", "ovg_match_workspace_bytes", "ovg_match_index",
                                         "ovg_match_query", "ovg_tracks_workspace_bytes", "ovg_tracks_assign",
                                         "ovg_tracks_gather"]
    _, a = dry.calls[5]
    assert a[2:6] == (max(P, 1), S, H * W, 1)
    assert dry.reads == 1
    assert out["points"].shape == (0, 3) and out["offsets"].shape == (1,) and out["view_offsets"].shape == (S + 1,)
    assert out["extrinsic"].shape == (S, 3, 4) and out["intrinsic"].shape == (S, 3, 3)


def test_errors_before_any_device_work(dry):
    from omnivggt_official_b200 import OmniVGGT
    pred = _scene(4, 6, 8)
    for mv in (0, 5, 2.0, True, None):
        with pytest.raises(ValueError, match="min_views"):
            OmniVGGT.tracks(pred, min_views=mv)
    with pytest.raises(ValueError, match="source"):
        OmniVGGT.tracks(pred, source="normals")
    with pytest.raises(ValueError, match="conf_percent"):
        OmniVGGT.tracks(pred, conf_percent=101.0)
    with pytest.raises(IndexError):
        OmniVGGT.tracks(pred, [(0, 4)])
    with pytest.raises(ValueError, match="itself"):
        OmniVGGT.tracks(pred, [(2, 2)])
    with pytest.raises(ValueError, match="mask_sky"):
        OmniVGGT.tracks(pred, mask_sky=torch.zeros(3, 6, 8, dtype=torch.bool))
    big = {"images": torch.empty(1, 2, 3, 32768, 32768, device="meta")}
    with pytest.raises(ValueError, match="2\\^31"):
        OmniVGGT.tracks(big)
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
def _np(d):
    return {k: v.cpu().numpy() for k, v in d.items() if torch.is_tensor(v)}


def _keep(pred, source="depth", pct=50.0, mask_sky=False):
    """The keep mask tracks() uses, on the host."""
    from omnivggt_official_b200 import OmniVGGT
    _, _, _, mask, _, _ = OmniVGGT._kept_views(pred, source, pct, 1e-5, None, 0, mask_sky)
    return mask.bool().cpu().numpy()


def _device_matches(pred, keep, pairs, source="depth", pct=50.0, mask_sky=False):
    """OmniVGGT.matches (pinned to matches_oracle by test_matches) in the oracle's kept-index layout."""
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = keep.shape
    rank = np.cumsum(keep.reshape(S, -1), 1) - 1
    pairs = [tuple(p) for p in TO.normalize_pairs(pairs, S).tolist()]
    out = OmniVGGT.matches(pred, pairs, source=source, conf_percent=pct, mask_sky=mask_sky) if pairs else []
    res = {}
    for (i, j), o in zip(pairs, out):
        xi, xj = o["xy_i"].cpu().numpy(), o["xy_j"].cpu().numpy()
        res[(i, j)] = (rank[i][xi[:, 1] * W + xi[:, 0]], rank[j][xj[:, 1] * W + xj[:, 0]])
    return res


def _oracle(pred, got, pairs, min_views, source="depth", pct=50.0, mask_sky=False, matches="device"):
    key = "world_points_from_depth" if source == "depth" else "world_points"
    keep = _keep(pred, source, pct, mask_sky)
    if matches == "device":
        matches = _device_matches(pred, keep, pairs, source, pct, mask_sky)
    elif matches == "kdtree":
        matches = None
    pts = pred[key][0].float().cpu().numpy()
    return TO.scene_tracks(pts, keep, pred["images"][0].float().cpu().numpy(), got["extrinsic"].cpu().numpy(),
                           got["intrinsic"].cpu().numpy(), pairs, min_views, nn=MO.nn_kdtree, matches=matches)


def _assert_equal(got, want):
    g = _np(got)
    for k in INT_KEYS + ("points", "error"):
        assert g[k].dtype == want[k].dtype or k in ("colors",), (k, g[k].dtype, want[k].dtype)
        assert g[k].shape == want[k].shape and np.array_equal(g[k], want[k]), k
        if g[k].dtype == np.float64:
            assert g[k].tobytes() == want[k].tobytes(), k


def _gpu_scene(S, H, W, seed=5):
    pred = _scene(S, H, W, seed)
    return {k: v.cuda() for k, v in pred.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("min_views", [1, 2, 3])
def test_surface_views_518_all_pairs(min_views):
    from omnivggt_official_b200 import OmniVGGT
    pred = _gpu_scene(8, 518, 518, seed=9)
    got = OmniVGGT.tracks(pred, min_views=min_views)
    want = _oracle(pred, got, None, min_views)
    assert len(want["points"]) > 1000 and (np.diff(want["offsets"]) >= min_views).all()
    _assert_equal(got, want)


@pytest.mark.gpu
def test_24_views_ranking_pairs():
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.geometry import compute_ranking
    pred = _gpu_scene(24, 60, 80, seed=3)
    ext = torch.eye(4)[None].repeat(24, 1, 1)
    ext[:, :3, 3] = torch.stack([torch.linspace(0, 3, 24), torch.sin(torch.linspace(0, 6, 24)), torch.zeros(24)], 1)
    ranking, _ = compute_ranking(ext.cuda(), k=8)
    pairs = [(i, int(r)) for i, row in enumerate(ranking.cpu().tolist()) for r in row if r != i]
    assert len(TO.normalize_pairs(pairs, 24)) < len(pairs)                  # reversed duplicates are merged
    for min_views in (2, 3):
        got = OmniVGGT.tracks(pred, pairs, min_views=min_views, conf_percent=30.0)
        _assert_equal(got, _oracle(pred, got, pairs, min_views, pct=30.0))


@pytest.mark.gpu
def test_mask_sky_and_pointmap():
    from omnivggt_official_b200 import OmniVGGT
    from test_sky import _blob_images
    pred = _gpu_scene(4, 64, 80, seed=2)
    pred["images"] = _blob_images(4, 64, 80, seed=2)[None].cuda()
    pred["world_points"] = pred["world_points_from_depth"] * 1.5
    pred["world_points_conf"] = pred["depth_conf"].flip(-1).contiguous()
    got = OmniVGGT.tracks(pred, mask_sky=True, conf_percent=10.0)
    want = _oracle(pred, got, None, 2, pct=10.0, mask_sky=True)
    assert 0 < len(want["points"])
    _assert_equal(got, want)
    got = OmniVGGT.tracks(pred, [(2, 0), (1, 3), (0, 2)], source="pointmap", min_views=1)
    _assert_equal(got, _oracle(pred, got, [(2, 0), (1, 3), (0, 2)], 1, source="pointmap"))


@pytest.mark.gpu
def test_end_to_end_against_ckdtree_matches():
    from omnivggt_official_b200 import OmniVGGT
    pred = _gpu_scene(3, 120, 160, seed=4)
    pred["world_points_from_depth"][0, 1, :, ::7] = pred["world_points_from_depth"][0, 1, :, 1::7]   # exact ties
    got = OmniVGGT.tracks(pred, min_views=2)
    _assert_equal(got, _oracle(pred, got, None, 2, matches="kdtree"))


@pytest.mark.gpu
def test_repeatable_and_independent_of_poisoned_memory():
    from omnivggt_official_b200 import OmniVGGT
    from test_poison_gpu import check_case
    pred = _gpu_scene(5, 48, 64, seed=6)
    a, b = OmniVGGT.tracks(pred, min_views=1), OmniVGGT.tracks(pred, min_views=1)
    for k in a:
        assert torch.equal(a[k].view(-1).view(torch.uint8), b[k].view(-1).view(torch.uint8)), k
    want = _oracle(pred, a, None, 2)
    check_case("tracks", lambda P: OmniVGGT.tracks(pred, min_views=2), finite=("points",),
               reference=lambda o: _assert_equal(o, want))


@pytest.mark.gpu
def test_non_finite_kept_point_raises():
    from omnivggt_official_b200 import OmniVGGT
    pred = _gpu_scene(3, 20, 24)
    pred["depth_conf"][0, 2, 5, 5] = 100.0
    pred["world_points_from_depth"][0, 2, 5, 5, 1] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        OmniVGGT.tracks(pred, conf_percent=0.0)
    with pytest.raises(ValueError, match="finite"):
        OmniVGGT.tracks(pred, [], conf_percent=0.0, min_views=1)
    pred["depth_conf"][0, 2, 5, 5] = 0.0                                   # dropped by the confidence floor
    assert len(OmniVGGT.tracks(pred, conf_percent=0.0)["points"]) > 0


@pytest.mark.gpu
def test_depth_consistent_points_reproject_onto_their_pixel_centres(tmp_path):
    """Points unprojected from depth with the cameras, one observation each: the error is ~0, so the writer's (x + 0.5,
    cx + 0.5) convention is that of the unprojection."""
    from omnivggt_official_b200 import OmniVGGT, ops
    from omnivggt_official_b200.colmap import write_colmap
    S, H, W = 3, 40, 56
    g = torch.Generator().manual_seed(1)
    pose = torch.cat([torch.randn(S, 3, generator=g) * 0.2, torch.nn.functional.normalize(
        torch.tensor([[0.05, -0.02, 0.01, 1.0]]) + 0.05 * torch.randn(S, 4, generator=g), dim=1),
        torch.full((S, 2), 1.0)], 1).cuda()
    ext, intr, c2w = ops.pose_decode(pose, H, W)
    depth = (2.0 + torch.rand(S, H, W, generator=g)).cuda()
    pred = {"images": torch.rand(1, S, 3, H, W, generator=g).cuda(), "extrinsic": ext[None], "intrinsic": intr[None],
            "world_points_from_depth": ops.unproject_depth(depth, intr, c2w, H, W)[None],
            "depth_conf": torch.ones(1, S, H, W).cuda()}
    out = OmniVGGT.tracks(pred, [], min_views=1, conf_percent=0.0)
    assert len(out["points"]) == S * H * W and float(out["error"].max()) <= 1e-3
    _assert_equal(out, _oracle(pred, out, [], 1, pct=0.0))
    cams, _, pts = TO.check_model(write_colmap(str(tmp_path), pred, out, images=False), True, ext.cpu().numpy(), H, W)
    assert cams[0][4][2] == float(intr[0, 0, 2]) + 0.5 and len(pts) == S * H * W


def _check_written(tmp_path, pred, out, S, H, W):
    from omnivggt_official_b200.colmap import write_colmap
    for binary in (True, False):
        folder = write_colmap(str(tmp_path / str(binary)), pred, out, binary=binary)
        cams, ims, pts = TO.check_model(folder, binary, out["extrinsic"].cpu().numpy(), H, W)
        assert len(cams) == len(ims) == S and len(pts) == len(out["points"]) > 0
        assert sorted(os.listdir(tmp_path / str(binary) / "images")) == [f"{i:06d}.png" for i in range(S)]
    assert TO.read_model(str(tmp_path / "True" / "sparse" / "0"), True) == TO.read_model(str(tmp_path / "False" / "sparse" / "0"),
                                                                                         False)


@pytest.mark.gpu
def test_mini_model_forward_export(tmp_path):
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
    raw = m(depth_gt_index=[1], camera_gt_index=[0], **inp)
    out = m.tracks(dict(raw), conf_percent=25.0)                       # cameras decoded from pose_enc inside
    pred = m.postprocess(raw)
    again = m.tracks(pred, conf_percent=25.0)
    assert torch.equal(out["extrinsic"], pred["extrinsic"][0]) and torch.equal(out["points"], again["points"])
    _assert_equal(out, _oracle(pred, out, None, 2, pct=25.0))
    _check_written(tmp_path, pred, out, 3, 56, 56)


@pytest.mark.gpu
def test_reconstruct_export(tmp_path):
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 10, 56, 56, seed=63).items()}
    rec = m.reconstruct(**inp, chunk=6, overlap=2)
    out = m.tracks(rec, min_views=3, conf_percent=25.0)
    assert torch.equal(out["extrinsic"], rec["extrinsic"][0])
    _assert_equal(out, _oracle(rec, out, None, 3, pct=25.0))
    _check_written(tmp_path, rec, out, 10, 56, 56)
