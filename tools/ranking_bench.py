"""Image ranking by camera distance on the device (libovg ovg_compute_ranking through geometry.compute_ranking) against the
reference's host computation (image_ranking.py:118-140) restated in numpy (oracle/ranking_oracle.py reference_numpy).

Views: seeded random poses with a dense video trajectory through every fifth view.  Sizes: 2 000 and 6 000 views (fp64
dists), 6 001 and 20 000 (the reference's fp32 chunked path), and 8 192 / 8 193 on each side of the shared-memory threshold
(OVG_RANK_CTA_VIEWS), each with k = None (the full [N, N] ranking) and k = 64.  Device: CUDA events around whole calls after
a warm-up, median of --reps.  Host: one call of the numpy restatement on this machine's CPUs, up to --host-max views (the
restatement's time grows as N^2: about 1 s at 2 000 views and 6 s at 6 000).  Every device result is checked: ranking equal
to torch.argsort(dists, stable=True), and 64 sampled rows of dists within 4 ulp of the oracle's fp64 truth.
        python tools/ranking_bench.py [--reps 5] [--host-max 6001]"""
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


def views(N, seed=0):
    from oracle.make_golden_ranking import poses, trajectory
    E = poses(np.random.default_rng(seed), N, np.float64)
    E[::5] = trajectory(len(E[::5]), np.float64)
    return E


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
    ap.add_argument("--host-max", type=int, default=6001)
    args = ap.parse_args()
    from omnivggt_official_b200.geometry import compute_ranking
    from oracle import ranking_oracle as RO
    rows = []
    for N in (2000, 6000, 6001, 8192, 8193, 20000):
        E = views(N, seed=N)
        ext = torch.from_numpy(E).cuda()
        full_ms, (ranking, dists) = _events(lambda: compute_ranking(ext), args.reps)
        top_ms, (top, _) = _events(lambda: compute_ranking(ext, k=64), args.reps)
        sample = np.sort(np.random.default_rng(N).choice(N, 64, replace=False))
        tr = RO.truth(E, rows=sample)
        row = {"N": N, "path": "smem" if N <= 8192 else "grid", "dists": str(dists.dtype).replace("torch.", ""),
               "device_ms": round(full_ms, 3), "device_k64_ms": round(top_ms, 3),
               "self_consistent": bool(torch.equal(ranking, torch.argsort(dists, dim=1, stable=True))),
               "equal_to_oracle": bool(RO.within_ulps(dists[torch.from_numpy(sample).cuda()].cpu().numpy(), tr).all()),
               "k64_equal": bool(torch.equal(top, ranking[:, :64]))}
        del ranking, dists, top
        torch.cuda.empty_cache()
        if N <= args.host_max:
            a = time.perf_counter()
            RO.reference_numpy(E)
            row["host_numpy_ms"] = round(1e3 * (time.perf_counter() - a), 1)
            row["speedup"] = round(row["host_numpy_ms"] / full_ms, 1)
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "cpus": os.cpu_count(),
                      "rows": rows}))


if __name__ == "__main__":
    main()
