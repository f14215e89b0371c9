"""Reciprocal nearest-neighbour matches (reference omnivggt/utils/geometry.py:435-451 find_reciprocal_matches).
CPU: the numpy oracle against the UNMODIFIED reference's outputs on a seeded case matrix (tests/golden/matches.json), the
large-set oracle against the definition, a dry run of the library calls, and the errors.
GPU: libovg's ovg_match_* against the oracle bit for bit, against cKDTree on two 518^2 views, a 24-view scene against per-pair
calls, and OmniVGGT.matches on the mini model."""
import hashlib
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import matches_oracle as MO
from oracle.make_golden_matches import make_cases, surface_views

GOLD = json.load(open(os.path.join(GOLDEN, "matches.json")))
CASES = make_cases()
NAMES = sorted(CASES)


def _sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _check_against_golden(name, rec, nn2, count):
    """Tie-free cases: bit for bit.  Cases with ties: the distances of the chosen neighbours (cKDTree's pick among ties is
    unspecified)."""
    g = GOLD[name]
    P1, P2 = CASES[name]
    assert (len(rec), len(nn2)) == (g["m"], g["m"])
    assert _sha(np.sqrt(MO.d2_of(P2, P1, nn2))) == g["dist2_sha256"]
    if not g["has_ties"]:
        assert count == g["count"]
        assert _sha(np.asarray(rec, bool)) == g["reciprocal_sha256"] and _sha(np.asarray(nn2, np.int64)) == g["nn2_in_P1_sha256"]


def _scene(S, H, W, seed=5):
    """Predictions of one scene: surface-like point maps, confidences with ties, images."""
    pts = surface_views(S, H, W, seed)
    g = torch.Generator().manual_seed(seed)
    conf = 1.0 + torch.rand(S, H, W, generator=g) * 4.0
    conf[..., ::6] = conf[0, 0, 0]
    return {"images": torch.rand(1, S, 3, H, W, generator=g), "world_points_from_depth": torch.from_numpy(pts)[None],
            "depth_conf": conf[None], "extrinsic": torch.eye(4)[:3].repeat(1, S, 1, 1)}


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_golden(name):
    P1, P2 = CASES[name]
    rec, nn2, count = MO.find_reciprocal_matches(P1, P2)
    _check_against_golden(name, rec, nn2, count)
    nn1, _ = MO.nn_brute(P1, P2)
    assert _sha(np.sqrt(MO.d2_of(P1, P2, nn1))) == GOLD[name]["dist1_sha256"]


@pytest.mark.parametrize("name", ["duplicates", "all_equal_same", "surface", "point_cloud_01", "far_outlier"])
def test_kdtree_oracle_equals_definition(name):
    P1, P2 = CASES[name]
    for Q, T in ((P1, P2), (P2, P1)):
        a, da = MO.nn_brute(Q, T)
        b, db = MO.nn_kdtree(Q, T)
        assert np.array_equal(a, b) and np.array_equal(da, db)


@pytest.fixture()
def dry(monkeypatch):
    """The C library replaced by a recorder, on CPU tensors; host reads counted."""
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
        return t.cpu()

    monkeypatch.setattr(_lib, "lib", lambda: rec)
    monkeypatch.setattr(_lib, "stream", lambda: 0)
    monkeypatch.setattr(ops, "_on_device", lambda t: True)
    monkeypatch.setattr(ops, "host_read", read)
    return rec


@pytest.mark.parametrize("pairs", [[(0, 1)], [(3, 1), (0, 2)], None])
def test_dry_run_builds_once_and_reads_once(dry, pairs):
    """One index build over all S views, one query call for all pairs, the same calls whatever the number of pairs, one read."""
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = 6, 8, 10
    out = OmniVGGT.matches(_scene(S, H, W), pairs)
    P = len(pairs) if pairs is not None else S * (S - 1) // 2
    assert [n for n, _ in dry.calls] == ["ovg_conf_percentile_mask", "ovg_match_workspace_bytes", "ovg_match_index",
                                         "ovg_match_query"]
    _, idx = dry.calls[2]
    assert idx[2:5] == (S, H * W, P)
    _, q = dry.calls[3]
    assert q[1:4] == (P, S, H * W)
    assert dry.reads == 1
    assert len(out) == P and all(o["count"] == 0 for o in out)


def test_errors_before_any_device_work(dry):
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.geometry import find_reciprocal_matches
    pred = _scene(4, 6, 8)
    with pytest.raises(ValueError, match="source"):
        OmniVGGT.matches(pred, source="normals")
    for pct in (-1.0, 100.5):
        with pytest.raises(ValueError, match="conf_percent"):
            OmniVGGT.matches(pred, conf_percent=pct)
    with pytest.raises(IndexError):
        OmniVGGT.matches(pred, [(0, 4)])
    with pytest.raises(IndexError):
        OmniVGGT.matches(pred, [(-1, 2)])
    with pytest.raises(ValueError, match="itself"):
        OmniVGGT.matches(pred, [(1, 2), (2, 2)])
    with pytest.raises(ValueError):
        OmniVGGT.matches(pred, [(1, 2, 3)])
    with pytest.raises(ValueError, match="shape"):
        find_reciprocal_matches(np.zeros((5, 2)), np.zeros((4, 3)))
    with pytest.raises(ValueError, match="shape"):
        find_reciprocal_matches(np.zeros((5, 3)), np.zeros((4, 3, 1)))
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
def _device_matches(P1, P2):
    from omnivggt_official_b200.geometry import find_reciprocal_matches
    rec, nn2, count = find_reciprocal_matches(torch.from_numpy(P1).cuda(), torch.from_numpy(P2).cuda())
    assert rec.is_cuda and rec.dtype == torch.bool and nn2.dtype == torch.int64 and isinstance(count, int)
    return rec.cpu().numpy(), nn2.cpu().numpy(), count


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_equals_oracle(name):
    P1, P2 = CASES[name]
    rec, nn2, count = _device_matches(P1, P2)
    orec, onn2, ocount = MO.find_reciprocal_matches(P1, P2)
    assert np.array_equal(rec, orec) and np.array_equal(nn2, onn2) and count == ocount
    _check_against_golden(name, rec, nn2, count)
    rec_b, nn2_b, count_b = _device_matches(P1, P2)                       # repeated calls are bit-identical
    assert np.array_equal(rec, rec_b) and np.array_equal(nn2, nn2_b) and count == count_b


@pytest.mark.gpu
def test_device_edge_cases():
    from omnivggt_official_b200.geometry import find_reciprocal_matches
    P = np.random.default_rng(0).random((100, 3)).astype(np.float32)
    for a, b in ((P[:0], P), (P, P[:0])):
        rec, nn2, count = find_reciprocal_matches(a, b)                   # arrays are moved to the device
        assert count == 0 and rec.shape == (len(b),) and not rec.any() and rec.is_cuda
    bad = P.copy()
    bad[7, 1] = np.nan
    for a, b in ((bad, P), (P, bad), (bad, bad), (P, np.full((5, 3), np.nan, np.float32)), (np.full((5, 3), np.nan, np.float32), P)):
        with pytest.raises(ValueError, match="finite"):
            find_reciprocal_matches(a, b)
    bad[7, 1] = np.inf
    for a, b in ((bad, P), (P, bad)):
        with pytest.raises(ValueError, match="finite"):
            find_reciprocal_matches(a, b)
    rec, nn2, count = find_reciprocal_matches(P, P)                       # the library is still usable after the errors
    assert count == 100
    rec, nn2, count = find_reciprocal_matches(P.astype(np.float64), P)    # used as fp32; every point is its own match
    assert count == 100 and np.array_equal(nn2.cpu().numpy(), np.arange(100))


@pytest.mark.gpu
def test_two_518_views_against_ckdtree():
    """About 268 k points per view: equal d2 everywhere, equal indices where there is no tie, the lowest index where there is."""
    from scipy.spatial import cKDTree
    sv = surface_views(2, 518, 518, seed=9)
    P1, P2 = sv[0].reshape(-1, 3), sv[1].reshape(-1, 3)
    P2[::1000] = P2[1::1000]                                               # duplicates: exact ties
    rec, nn2, count = _device_matches(P1, P2)
    dist, kd = cKDTree(P1).query(P2, workers=-1)
    assert np.array_equal(np.sqrt(MO.d2_of(P2, P1, nn2)), dist)
    onn2, _ = MO.nn_kdtree(P2, P1)
    assert np.array_equal(nn2, onn2)
    orec, _, ocount = MO.find_reciprocal_matches(P1, P2, nn=MO.nn_kdtree)
    assert np.array_equal(rec, orec) and count == ocount
    assert (nn2 != kd).sum() <= (MO.d2_of(P2, P1, kd) == MO.d2_of(P2, P1, nn2)).sum()


@pytest.mark.gpu
def test_scene_all_pairs_equal_per_pair_calls():
    """S = 24: every pair of one batched call equals find_reciprocal_matches on the kept points of the two views; the call's
    kernel launches do not depend on the number of pairs."""
    from omnivggt_official_b200 import OmniVGGT, _lib, ops
    from omnivggt_official_b200.geometry import find_reciprocal_matches
    S, H, W = 24, 30, 40
    pred = {k: v.cuda() for k, v in _scene(S, H, W).items()}
    lib = _lib.load()
    n0 = lib.ovg_launch_count()
    OmniVGGT.matches(pred, [(3, 5)], conf_percent=30.0)
    n1 = lib.ovg_launch_count()
    out = OmniVGGT.matches(pred, conf_percent=30.0)
    n2 = lib.ovg_launch_count()
    assert len(out) == S * (S - 1) // 2 and n2 - n1 == n1 - n0
    mask, _, _ = ops.conf_percentile_mask(pred["depth_conf"][0].contiguous(), 30.0, 1e-5)
    keep = mask.bool().view(S, -1)
    pts = pred["world_points_from_depth"][0].reshape(S, -1, 3)
    grid = torch.from_numpy(MO.xy_grid(W, H).reshape(-1, 2)).cuda()
    pairs = [(i, j) for i in range(S) for j in range(i + 1, S)]
    for (i, j), o in zip(pairs, out):
        rec, nn2, count = find_reciprocal_matches(pts[i][keep[i]], pts[j][keep[j]])
        assert o["count"] == count > 0
        assert torch.equal(o["xy_j"], grid[keep[j]][rec]) and torch.equal(o["xy_i"], grid[keep[i]][nn2][rec])
    again = OmniVGGT.matches(pred, conf_percent=30.0)
    for a, b in zip(out, again):
        assert torch.equal(a["xy_i"], b["xy_i"]) and torch.equal(a["xy_j"], b["xy_j"])
    # the whole scene against the numpy oracle on the same keep mask
    ref = MO.scene_matches(pts.cpu().numpy().reshape(S, H, W, 3), keep.cpu().numpy().reshape(S, H, W), pairs[:40])
    for o, r in zip(out, ref):
        assert o["count"] == r["count"] and np.array_equal(o["xy_i"].cpu().numpy(), r["xy_i"])
        assert np.array_equal(o["xy_j"].cpu().numpy(), r["xy_j"])


@pytest.mark.gpu
def test_scene_with_non_finite_kept_points_raises():
    """A NaN kept point in view j of a pair, or a view whose kept points are all NaN, raises after the read; a NaN pixel that
    the confidence mask drops does not."""
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = 4, 20, 24
    base = _scene(S, H, W)
    base["depth_conf"][0, :, 0, 0] = 0.0                                  # pixel (0, 0) is never kept
    for view, where in ((2, (3, 4)), (1, (0, 0)), (3, slice(None))):
        pred = {k: v.clone().cuda() for k, v in base.items()}
        pred["world_points_from_depth"][0, view][where] = float("nan")
        if view == 1:
            OmniVGGT.matches(pred, [(0, 1)], conf_percent=0.0)
            continue
        with pytest.raises(ValueError, match="finite"):
            OmniVGGT.matches(pred, [(0, view)], conf_percent=0.0)
        with pytest.raises(ValueError, match="finite"):
            OmniVGGT.matches(pred, [(view, 0)], conf_percent=0.0)
    assert OmniVGGT.matches({k: v.cuda() for k, v in base.items()}, [(0, 1)], conf_percent=0.0)[0]["count"] > 0


@pytest.mark.gpu
def test_identical_views_match_every_pixel_to_itself():
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = 3, 40, 52
    pred = _scene(S, H, W)
    wp = pred["world_points_from_depth"]
    wp[0, 2] = wp[0, 0]
    wp[0, 0, 5, 7] = wp[0, 0, 5, 6]                                        # one duplicate pair inside the view
    pred = {k: v.cuda() for k, v in pred.items()}
    pred["depth_conf"][0, 2] = pred["depth_conf"][0, 0]
    o = OmniVGGT.matches(pred, [(0, 2)], conf_percent=0.0)[0]
    assert o["count"] == H * W - 1
    assert torch.equal(o["xy_i"], o["xy_j"])
    assert not ((o["xy_j"][:, 0] == 7) & (o["xy_j"][:, 1] == 5)).any()     # the later duplicate matches the earlier one


@pytest.mark.gpu
def test_model_matches_api():
    from test_model_gpu import model
    from omnivggt_official_b200 import ops
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
    raw = m(depth_gt_index=[1], camera_gt_index=[0], **inp)
    pred = m.postprocess(raw)
    for source in ("depth", "pointmap"):
        out = m.matches(pred, source=source, conf_percent=25.0)
        assert len(out) == 3
        key, ckey = ("world_points_from_depth", "depth_conf") if source == "depth" else ("world_points", "world_points_conf")
        mask, _, _ = ops.conf_percentile_mask(pred[ckey][0].float().contiguous(), 25.0, 1e-5)    # the mask matches() uses
        keep = mask.bool().cpu().numpy()
        ref = MO.scene_matches(pred[key][0].float().cpu().numpy(), keep, [(0, 1), (0, 2), (1, 2)])
        for o, r in zip(out, ref):
            assert o["count"] == r["count"]
            assert np.array_equal(o["xy_i"].cpu().numpy(), r["xy_i"]) and np.array_equal(o["xy_j"].cpu().numpy(), r["xy_j"])
            assert o["xy_i"].shape == (o["count"], 2) and o["xy_i"].dtype == torch.int64
    direct = m.matches(dict(raw), [(2, 0)])                                 # unprojected inside when postprocess() has not run
    assert direct[0]["xy_i"].shape[1] == 2
