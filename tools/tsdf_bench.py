"""Fused mesh on the device (OmniVGGT.fused_mesh: libovg ovg_tsdf_*) on synthetic scenes of 8 and 24 views at 518^2 (exact
depth maps of a sphere and a box seen from a ring of cameras, tests/test_fused_mesh.py) at resolutions 256 and 512.

Per phase, CUDA events around each library call after a warm-up of every shape, median over --reps calls:
  bounds     ovg_tsdf_bounds (1st / 99th percentiles of the kept points; the kept mask and cameras are built once, outside)
  integrate  ovg_tsdf_integrate (brick marking and integration)
  count      ovg_tsdf_count
  extract    ovg_tsdf_extract
and the whole OmniVGGT.fused_mesh call (two host reads included) by perf_counter around a synchronised call.  Also the grid,
the marked-brick fraction, the vertex and triangle counts, and one check of the whole result against the numpy oracle
(oracle/tsdf_oracle.py), with the GPU name and power limit.
        python tools/tsdf_bench.py [--reps 10] [--no-oracle]"""
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def _events(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return round(ts[len(ts) // 2], 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-oracle", action="store_true")
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT, ops
    from omnivggt_official_b200 import scene as SC
    from oracle import tsdf_oracle as TO
    from test_fused_mesh import assert_equal_to_oracle, oracle_of, synthetic_scene
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "sizes": []}
    checked = args.no_oracle
    for S in (8, 24):
        pred = {k: v.cuda() for k, v in synthetic_scene("two", S, 518, 518, seed=S).items()}
        images, (ext, intr), points, mask, _, _ = SC._kept_views(pred, "depth", 10.0, 1e-5, None, 0, False,
                                                                cameras="predictions")
        depth = pred["depth"][0, ..., 0].contiguous()
        for resolution in (256, 512):
            b = ops.tsdf_bounds(points, mask).cpu().numpy()
            origin, s, trunc, shape = SC._fusion_grid(b[1:4], b[4:7], resolution)
            ws = ops.tsdf_workspace(points.device, shape)
            vol = {}

            def integrate():
                vol["t"], vol["c"] = ops.tsdf_integrate(depth, mask, images, ext, intr, shape, origin, s, trunc, ws)

            def count():
                vol["mc"] = ops.TsdfMesher(vol["t"], origin, s, ws)

            integrate()
            count()
            m, k = vol["mc"].totals.tolist()

            def extract():
                vol["mc"].extract(vol["c"], m, k)

            phases = {"bounds_ms": lambda: ops.tsdf_bounds(points, mask), "integrate_ms": integrate, "count_ms": count,
                      "extract_ms": extract}
            row = {"views": S, "pixels": S * 518 * 518, "resolution": resolution, "grid": list(shape)}
            for name, fn in phases.items():
                fn()
                row[name] = _events(fn, args.reps)
            OmniVGGT.fused_mesh(pred, resolution=resolution, conf_percent=10.0)
            ts = []
            for _ in range(args.reps):
                torch.cuda.synchronize()
                a = time.perf_counter()
                OmniVGGT.fused_mesh(pred, resolution=resolution, conf_percent=10.0)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - a)
            row["fused_mesh_ms"] = round(1e3 * sorted(ts)[len(ts) // 2], 2)
            bricks = np.prod([(n + 7) // 8 for n in shape])
            live = (~torch.isnan(vol["t"])).sum().item()
            row.update(vertices=m, triangles=k, bricks=int(bricks), observed_voxels=int(live),
                       workspace_bytes=int(ws.numel()))
            if not checked:
                want = oracle_of(pred, resolution)
                res_, t_, c_ = SC._fusion(pred, resolution, 10.0, 1e-5, 0, False)
                assert_equal_to_oracle(res_, t_, c_, want)
                row["oracle_equal"] = True
                checked = True
            mk = TO.mark_bricks(depth.cpu().numpy(), mask.cpu().numpy(), ext.cpu().numpy(), intr.cpu().numpy(),
                                origin, s, trunc, shape[::-1])          # the device's marks: its volume equals the oracle's
            row["marked_fraction"] = round(float(mk.mean()), 4)
            res["sizes"].append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
