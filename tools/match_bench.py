"""Reciprocal nearest-neighbour matches on the device (OmniVGGT.matches / geometry.find_reciprocal_matches: libovg ovg_match_*)
against the reference's host path (utils/geometry.py:435-451: two cKDTree builds and queries per pair, here with workers = the
host's CPUs) on the same inputs, outputs checked equal.

Workloads: all pairs of 8 and of 24 seeded surface-like 518^2 views at conf_percent=50; one find_reciprocal_matches of two
518^2 views (268 k x 268 k points); the same with one far outlier in P1.  Device: CUDA events over repeated calls after a
warm-up, including the one host read of each call.        python tools/match_bench.py [--reps 5]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import matches_oracle as MO  # noqa: E402
from oracle.make_golden_matches import surface_views  # noqa: E402


def host_find_reciprocal_matches(P1, P2):
    """geometry.py:442-451 with workers = the host's CPUs."""
    from scipy.spatial import cKDTree
    tree1, tree2 = cKDTree(P1), cKDTree(P2)
    _, nn1_in_P2 = tree2.query(P1, workers=os.cpu_count())
    _, nn2_in_P1 = tree1.query(P2, workers=os.cpu_count())
    reciprocal_in_P2 = nn1_in_P2[nn2_in_P1] == np.arange(len(nn2_in_P1))
    return reciprocal_in_P2, nn2_in_P1, reciprocal_in_P2.sum()


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        out = fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps, out


def scene(S, H=518, W=518, seed=0):
    pts = torch.from_numpy(surface_views(S, H, W, seed))[None].cuda()
    g = torch.Generator(device="cuda").manual_seed(seed)
    conf = 1.0 + torch.rand(1, S, H, W, device="cuda", generator=g) * 4.0
    return {"images": torch.zeros(1, S, 3, H, W, device="cuda"), "world_points_from_depth": pts, "depth_conf": conf,
            "extrinsic": torch.eye(4, device="cuda")[:3].repeat(1, S, 1, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT, ops
    from omnivggt_official_b200.geometry import find_reciprocal_matches
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cpus": os.cpu_count(), "rows": []}
    print(json.dumps({k: res[k] for k in ("gpu", "power_limit", "host_cpus")}), flush=True)
    for S in (8, 24):
        pred = scene(S)
        dev_ms, out = timed(lambda: OmniVGGT.matches(pred, conf_percent=50.0), args.reps)
        mask, _, _ = ops.conf_percentile_mask(pred["depth_conf"][0].contiguous(), 50.0, 1e-5)
        keep = mask.bool().view(S, -1).cpu().numpy()
        pts = pred["world_points_from_depth"][0].reshape(S, -1, 3).cpu().numpy()
        grid = MO.xy_grid(518, 518).reshape(-1, 2)
        pairs = [(i, j) for i in range(S) for j in range(i + 1, S)]
        t = time.perf_counter()
        equal = True
        for (i, j), o in zip(pairs, out):
            rec, nn2, n = host_find_reciprocal_matches(pts[i][keep[i]], pts[j][keep[j]])
            equal &= int(n) == o["count"] and np.array_equal(grid[keep[j]][rec], o["xy_j"].cpu().numpy()) and \
                np.array_equal(grid[keep[i]][nn2][rec], o["xy_i"].cpu().numpy())
        host_s = time.perf_counter() - t         # includes the comparison, which is small next to the cKDTree work
        row = {"workload": f"matches, {S} views 518^2, all {len(pairs)} pairs", "points_per_view": int(keep.sum(1).mean()),
               "matches": int(sum(o["count"] for o in out)), "device_ms": round(dev_ms, 2), "host_ms": round(1e3 * host_s, 1),
               "equal": bool(equal)}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    sv = surface_views(2, 518, 518, seed=1)
    P1, P2 = sv[0].reshape(-1, 3), sv[1].reshape(-1, 3)
    far = P1.copy()
    far[1234] = (1e6, -2e6, 5e5)
    for name, a in (("find_reciprocal_matches 268k x 268k", P1), ("same, one far outlier in P1", far)):
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(P2).cuda()
        dev_ms, (rec, nn2, n) = timed(lambda: find_reciprocal_matches(da, db), args.reps)
        t = time.perf_counter()
        hrec, hnn2, hn = host_find_reciprocal_matches(a, P2)
        host_s = time.perf_counter() - t
        equal = int(hn) == n and np.array_equal(hrec, rec.cpu().numpy()) and np.array_equal(hnn2, nn2.cpu().numpy())
        row = {"workload": name, "points_per_view": len(a), "matches": n, "device_ms": round(dev_ms, 2),
               "host_ms": round(1e3 * host_s, 1), "equal": bool(equal)}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
