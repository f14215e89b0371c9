"""Farthest point sampling: the numpy oracle against the unmodified reference's farthest_point_sample (CPU), the call pattern
of the drop-in and of point_cloud(max_points=...) on a recorded library (CPU), and the libovg kernel against the oracles
on every path it takes (GPU)."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import fps_oracle as FO
from oracle.make_golden_fps import make_cases

CASES = make_cases()


def _gold():
    with open(os.path.join(GOLDEN, "fps.json")) as f:
        return json.load(f)


def _sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _seeded_start(k):
    """The start the reference draws for a deterministic=False case, from the same seed."""
    torch.manual_seed(k["seed"])
    B, N = k["xyz"].shape[:2]
    return torch.randint(0, N, (B,), dtype=torch.long)


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference_golden(name):
    g, k = _gold()[name], CASES[name]
    assert _sha(k["xyz"]) == g["xyz_sha256"], "make_cases no longer reproduces the input"
    start = None if k["deterministic"] else _seeded_start(k).numpy()
    idx = FO.farthest_point_sample(k["xyz"], k["npoint"], k["include_ends"], start)
    assert list(idx.shape) == g["inds_shape"] and idx.dtype == np.int64
    assert _sha(idx) == g["inds_sha256"]


def test_torch_restatement_matches_numpy_oracle_on_cpu():
    for name in ("b2", "include_ends", "lattice_duplicates", "nonfinite", "beyond_1e10", "float64"):
        k = CASES[name]
        a = FO.farthest_point_sample(k["xyz"], k["npoint"], k["include_ends"])
        t = FO.farthest_point_sample_torch(torch.from_numpy(k["xyz"]), k["npoint"], k["include_ends"])
        assert np.array_equal(a, t.numpy()), name


@pytest.fixture()
def dry(monkeypatch):
    """The C library replaced by a recorder, on CPU tensors; host reads counted.  The recorded sampler writes index 0."""
    from omnivggt_official_b200 import _lib, geometry, ops

    class Rec:
        def __init__(self):
            self.calls, self.reads, self.count = [], 0, 0

        def __getattr__(self, name):
            def fn(*a):
                self.calls.append((name, a))
                if name == "ovg_farthest_point_sample":
                    ctypes.memset(a[8], 0, a[1] * a[3] * 8)
                return 0
            return fn

    rec = Rec()

    def read(t):
        rec.calls.append(("host_read", ()))
        rec.reads += 1
        t = t.cpu().clone()
        t.view(-1)[0] = rec.count                            # the kept count of point_cloud
        return t

    monkeypatch.setattr(_lib, "lib", lambda: rec)
    monkeypatch.setattr(_lib, "stream", lambda: 0)
    monkeypatch.setattr(ops, "_on_device", lambda t: True)
    monkeypatch.setattr(ops, "host_read", read)
    monkeypatch.setattr(geometry, "_device_of", lambda *xs: torch.device("cpu"))
    return rec


def test_dry_run_drop_in_is_one_call_without_host_read(dry):
    from omnivggt_official_b200.geometry import farthest_point_sample
    xyz = torch.randn(3, 500, 3, dtype=torch.float64)
    for npoint in (1, 7, 500):
        for ends in (False, True):
            dry.calls.clear()
            idx = farthest_point_sample(xyz, npoint, include_ends=ends, deterministic=npoint == 7)
            assert [n for n, _ in dry.calls] == ["ovg_fps_workspace_bytes", "ovg_farthest_point_sample"]
            a = dry.calls[1][1]
            assert a[1:4] == (3, 500, npoint) and a[5] == int(ends)
            assert idx.shape == (3, npoint) and idx.dtype == torch.int64
    assert dry.reads == 0


def test_drop_in_draws_the_start_as_the_reference_does(dry, monkeypatch):
    """Same torch.manual_seed, same start (misc.py:127-130); deterministic draws randint(0, 1) as the reference does."""
    from omnivggt_official_b200 import geometry, ops
    seen = []
    monkeypatch.setattr(ops, "farthest_point_sample", lambda pts, n, start, ends: seen.append(start.clone()) or
                        torch.zeros(pts.shape[0], n, dtype=torch.int64))
    for det in (False, True):
        torch.manual_seed(5)
        geometry.farthest_point_sample(np.zeros((4, 1000, 3), np.float32), 3, deterministic=det)
        after = torch.rand(1)
        torch.manual_seed(5)
        want = torch.randint(0, 1 if det else 1000, (4,), dtype=torch.long)
        assert torch.equal(seen[-1], want) and torch.equal(torch.rand(1), after)


def _scene(S, H, W, seed=3):
    g = torch.Generator().manual_seed(seed)
    ext = torch.eye(4)[:3].repeat(1, S, 1, 1)
    return {"images": torch.rand(1, S, 3, H, W, generator=g), "world_points_from_depth": torch.randn(1, S, H, W, 3, generator=g),
            "depth_conf": 1.0 + torch.rand(1, S, H, W, generator=g), "extrinsic": ext}


def test_dry_run_point_cloud_max_points(dry):
    """max_points adds one sampler call after the gather when more points are kept, and no host read."""
    from omnivggt_official_b200 import OmniVGGT
    base = ["ovg_conf_percentile_mask", "ovg_point_cloud_workspace_bytes", "ovg_point_cloud_count", "ovg_point_cloud_center",
            "host_read", "ovg_point_cloud_gather"] + ["ovg_point_cloud_scale"]
    dry.count = 50
    for max_points, sampled in ((None, False), (50, False), (200, False), (49, True), (1, True), (10, True)):
        dry.calls.clear()
        dry.reads = 0
        out = OmniVGGT.point_cloud(_scene(2, 6, 8), max_points=max_points)
        names = [n for n, _ in dry.calls]
        assert names == base + (["ovg_fps_workspace_bytes", "ovg_farthest_point_sample"] if sampled else []), names
        assert dry.reads == 1
        n = max_points if sampled else 50
        assert out["points"].shape == (n, 3) and out["colors"].shape == (n, 3) and out["frame"].shape == (n,)
        if sampled:
            a = dry.calls[-1][1]
            assert a[1:4] == (1, 50, max_points) and a[5] == 0


def test_errors_before_any_library_call(dry):
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.geometry import farthest_point_sample
    for xyz, npoint, what in ((np.zeros((1, 10, 2)), 3, "shape"), (np.zeros((1, 10, 4)), 3, "shape"),
                              (np.zeros((10, 3)), 3, "shape"), (np.zeros((2, 0, 3)), 1, "no points"),
                              (np.zeros((1, 10, 3)), 0, "npoint"), (np.zeros((1, 10, 3)), -2, "npoint"),
                              (np.zeros((1, 10, 3)), 11, "npoint")):
        with pytest.raises(ValueError, match=what):
            farthest_point_sample(xyz, npoint)
    pred = _scene(2, 6, 8)
    for bad in (0, -1, 2.5, True, "10"):
        with pytest.raises((ValueError, TypeError), match="max_points"):
            OmniVGGT.point_cloud(pred, max_points=bad)
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_kernel_matches_golden(name):
    from omnivggt_official_b200.geometry import farthest_point_sample
    g, k = _gold()[name], CASES[name]
    start = None if k["deterministic"] else _seeded_start(k)
    if k["seed"] is not None:
        torch.manual_seed(k["seed"])
    idx = farthest_point_sample(torch.from_numpy(k["xyz"]).cuda(), k["npoint"], k["include_ends"], k["deterministic"])
    idx = idx.cpu().numpy()
    assert idx.dtype == np.int64 and list(idx.shape) == g["inds_shape"]
    assert _sha(idx) == g["inds_sha256"]
    o = FO.farthest_point_sample(k["xyz"], k["npoint"], k["include_ends"], None if start is None else start.numpy())
    assert np.array_equal(idx, o)


CTA = 14336          # OVG_FPS_CTA_POINTS: one CTA per batch up to here, the cooperative grid above


def _surface(S, H, W):
    from oracle.make_golden_matches import surface_views
    return torch.from_numpy(surface_views(S=S, H=H, W=W).reshape(1, -1, 3))


def _gauss(B, N, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, 3, generator=g)
    x[:, ::7] = torch.round(x[:, ::7] * 4) / 4                   # exact duplicates and ties
    return x


SIZES = {
    "cta_n1_b3": (lambda: _gauss(3, 1, 1), 1, False),
    "cta_b3_odd": (lambda: _gauss(3, 1001, 2), 300, False),
    "cta_threshold": (lambda: _gauss(1, CTA, 3), 2000, False),
    "cta_threshold_ends_b2": (lambda: _gauss(2, CTA, 4), 700, True),
    "grid_above_threshold": (lambda: _gauss(1, CTA + 1, 5), 2000, False),
    "grid_b3_odd": (lambda: _gauss(3, 100003, 6), 1024, True),
    "grid_more_batches_than_ctas": (lambda: _gauss(200, CTA + 5, 7), 40, False),
    "grid_streamed_surface_8x518": (lambda: _surface(8, 518, 518), 4096, False),
    "grid_streamed_b2": (lambda: _gauss(2, 2_500_001, 8), 512, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SIZES))
def test_kernel_matches_torch_restatement(name):
    """Every path: one CTA per batch, the grid with all points in shared memory, several batches per group of CTAs, and
    points streamed from global memory (8 x 518^2 = 2.1 M points and 2 x 2.5 M are above the grid's shared memory)."""
    from omnivggt_official_b200 import ops
    make, npoint, ends = SIZES[name]
    xyz = make().cuda().contiguous()
    B = xyz.shape[0]
    start = torch.randint(0, xyz.shape[1], (B,), generator=torch.Generator().manual_seed(9)).cuda()
    got = ops.farthest_point_sample(xyz, npoint, start, ends)
    want = FO.farthest_point_sample_torch(xyz, npoint, ends, start)
    assert torch.equal(got, want), (got != want).nonzero()[:5]


@pytest.mark.gpu
def test_runs_are_bit_identical():
    from omnivggt_official_b200 import ops
    xyz = _surface(8, 518, 518).cuda()
    start = torch.zeros(1, dtype=torch.int64, device="cuda")
    a = ops.farthest_point_sample(xyz, 4096, start)
    b = ops.farthest_point_sample(xyz, 4096, start)
    c = ops.farthest_point_sample(xyz[:, :CTA].contiguous(), 4096, start)
    d = ops.farthest_point_sample(xyz[:, :CTA].contiguous(), 4096, start)
    assert torch.equal(a, b) and torch.equal(c, d)


def _cuda_scene(S, H, W, seed):
    return {k: v.cuda() for k, v in _scene(S, H, W, seed).items()}


@pytest.mark.gpu
@pytest.mark.parametrize("S,H,W,m", [(3, 64, 80, 1000), (4, 128, 128, 4096)])
def test_point_cloud_max_points_is_the_sampled_full_cloud(S, H, W, m, tmp_path):
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.glb import write_glb
    from test_point_cloud import _parse_glb, _read_cloud
    pred = _cuda_scene(S, H, W, seed=S)
    pred["world_points_from_depth"][0, 0, :4] = 0.5               # repeated positions
    full = OmniVGGT.point_cloud(pred, mask_black_bg=True)
    n = len(full["points"])
    assert n > m
    sampled = OmniVGGT.point_cloud(pred, mask_black_bg=True, max_points=m)
    idx = torch.from_numpy(FO.farthest_point_sample(full["points"][None].cpu().numpy(), m)[0]).cuda()
    for k in ("points", "colors", "frame"):
        assert torch.equal(sampled[k], full[k][idx]), k
    for k in ("conf_threshold", "center", "scale", "align"):
        assert torch.equal(sampled[k], full[k]), k
    for big in (n, n + 1, 10 * n):
        same = OmniVGGT.point_cloud(pred, mask_black_bg=True, max_points=big)
        for k in full:
            assert torch.equal(same[k], full[k]), (big, k)
    path = tmp_path / "sampled.glb"
    write_glb(str(path), sampled)
    p, c = _read_cloud(*_parse_glb(path.read_bytes()))
    assert np.array_equal(p, sampled["points"].cpu().numpy()) and np.array_equal(c[:, :3], sampled["colors"].cpu().numpy())


@pytest.mark.gpu
def test_point_cloud_max_points_with_fewer_distinct_positions_repeats():
    """A cloud with fewer distinct positions than max_points repeats points, as the reference's indices do."""
    from omnivggt_official_b200 import OmniVGGT
    pred = _cuda_scene(1, 16, 16, seed=1)
    pred["world_points_from_depth"][:] = torch.tensor([1.0, 2.0, 3.0], device="cuda")
    pred["world_points_from_depth"][0, 0, 0, 0] = torch.tensor([0.0, 0.0, 0.0], device="cuda")
    full = OmniVGGT.point_cloud(pred, conf_percent=0.0)
    out = OmniVGGT.point_cloud(pred, conf_percent=0.0, max_points=5)
    idx = torch.from_numpy(FO.farthest_point_sample(full["points"][None].cpu().numpy(), 5)[0]).cuda()
    assert torch.equal(out["points"], full["points"][idx])
    assert len(torch.unique(out["points"], dim=0)) <= 2
