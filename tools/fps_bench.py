"""Farthest point sampling on the device (libovg ovg_farthest_point_sample through geometry.farthest_point_sample) against the
reference's algorithm (po_utils/misc.py:114-148) run by torch, on CUDA tensors on the same GPU and on the host CPU.

Points: surface-like point maps of 8 and 24 views at 518^2 with a seeded half of the pixels kept (1.07 M and 3.2 M points,
the first within the cooperative grid's shared memory on a 132-SM H100, the second partly streamed from L2), budgets of
16 384 and 100 000, and two sizes on each side of the one-CTA threshold (OVG_FPS_CTA_POINTS = 14 336).
Device: CUDA events around whole calls after a warm-up, median of --reps.  torch: oracle/fps_oracle.py's restatement of the
reference loop, one call timed after a warm-up; it uses torch.where where the reference assigns through a boolean mask
(distance[mask] = dist[mask], which synchronises with the host every step), so it is a lower bound on the reference's time.
Host CPU: the same restatement on CPU tensors at a reduced size (one view, 1 024 samples), perf_counter.  Every device result
is checked equal to the torch one.
        python tools/fps_bench.py [--reps 5]"""
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


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def kept_points(S, H=518, W=518, seed=0):
    """Surface-like points of S views with a seeded half kept: fp32 [1, n, 3]."""
    from oracle.make_golden_matches import surface_views
    pts = surface_views(S=S, H=H, W=W, seed=seed).reshape(-1, 3)
    keep = np.random.default_rng(seed).random(len(pts)) < 0.5
    return torch.from_numpy(np.ascontiguousarray(pts[keep]))[None]


def _events(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from omnivggt_official_b200.geometry import farthest_point_sample
    from oracle.fps_oracle import farthest_point_sample_torch
    sizes = [("1 view 160^2 half", kept_points(1, 160, 160), 4096),
             ("1 view 200^2 half", kept_points(1, 200, 200), 4096)]
    for S in (8, 24):
        pts = kept_points(S)
        sizes += [(f"{S} views 518^2 half", pts, 16384), (f"{S} views 518^2 half", pts, 100000)]
    rows = []
    for name, pts, npoint in sizes:
        xyz = pts.cuda()
        dev_ms, idx = _events(lambda: farthest_point_sample(xyz, npoint, deterministic=True), args.reps)
        farthest_point_sample_torch(xyz, min(npoint, 64))
        torch.cuda.synchronize()
        a = time.perf_counter()
        ref = farthest_point_sample_torch(xyz, npoint)
        torch.cuda.synchronize()
        torch_ms = 1e3 * (time.perf_counter() - a)
        row = {"points": name, "n": xyz.shape[1], "path": "cta" if xyz.shape[1] <= 14336 else "grid", "npoint": npoint,
               "device_ms": round(dev_ms, 3), "torch_cuda_ms": round(torch_ms, 1), "speedup": round(torch_ms / dev_ms, 1),
               "equal": bool(torch.equal(idx, ref))}
        rows.append(row)
        print(json.dumps(row), flush=True)
    host = kept_points(1)
    a = time.perf_counter()
    farthest_point_sample_torch(host, 1024)
    host_ms = 1e3 * (time.perf_counter() - a)
    hrow = {"points": "1 view 518^2 half", "n": host.shape[1], "npoint": 1024, "host_cpu_ms": round(host_ms, 1)}
    xyz = host.cuda()
    hrow["device_ms"] = round(_events(lambda: farthest_point_sample(xyz, 1024, deterministic=True), args.reps)[0], 3)
    print(json.dumps(hrow), flush=True)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "cpus": os.cpu_count(),
                      "rows": rows, "host": hrow}))


if __name__ == "__main__":
    main()
