"""Scene evaluation on the device (OmniVGGT.evaluate: libovg ovg_eval_*, with ovg_sim3_* and the matcher) against its fp64
oracle on the host (oracle/eval_oracle.py: numpy and scipy's cKDTree), on the seeded sphere scenes of tests/test_evaluate.py:
  24 views of 518^2   all three groups (pose, depth, points)
  300 and 1000 views  the pose group
Device: the whole evaluate call (its host reads included) by perf_counter around a synchronised call, median of --reps after a
warm-up.  Host: the oracle on the same arrays, once.  The GPU name and power limit are read in the same run.
        python tools/eval_bench.py [--reps 5]"""
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


def device_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT
    from oracle import eval_oracle as EO
    import test_evaluate as T

    if not torch.cuda.is_available():
        raise SystemExit("eval_bench needs a CUDA device")
    cuda = T._cuda
    rows = []
    # all three groups at 24 views of 518^2
    S, H, W = 24, 518, 518
    ext, intr, depth, pts, pred_ext = T._points_case(S, H, W, seed=24)
    pred = T._pred(S, H, W, extrinsic=cuda(pred_ext)[None], depth=cuda(depth * 0.5)[None], world_points_from_depth=cuda(pts)[None])
    gt = dict(extrinsics=cuda(ext)[None], intrinsics=cuda(intr)[None], depth=cuda(depth)[None])
    dev = device_time(lambda: OmniVGGT.evaluate(pred, **gt), args.reps)
    out = OmniVGGT.evaluate(pred, **gt)
    t0 = time.perf_counter()
    EO.pose_metrics(ext, intr, pred_ext)
    EO.depth_metrics(depth, (depth * 0.5).astype(np.float32))
    g, keep, aligned = T._device_clouds(ext, intr, depth, pts, out["points"]["sim3"].cpu().numpy())
    EO.umeyama(pts[keep], g[keep])
    EO.point_metrics(aligned, g, keep)
    host = time.perf_counter() - t0
    rows.append({"case": f"all groups, {S} views {H}x{W}", "points": int(out["points"]["pixels"]), "device_s": dev,
                 "host_oracle_s": host, "chamfer": float(out["points"]["chamfer"]), "abs_rel": float(out["depth"]["abs_rel"])})
    # the pose group alone
    for n in (300, 1000):
        e, k, p = T._pose_case(n, seed=n)
        predp = T._pred(n, 4, 4, extrinsic=cuda(p)[None])
        gtp = dict(extrinsics=cuda(e)[None], intrinsics=cuda(k)[None])
        dev = device_time(lambda: OmniVGGT.evaluate(predp, **gtp), args.reps)
        t0 = time.perf_counter()
        EO.pose_metrics(e, k, p)
        rows.append({"case": f"pose, {n} views ({n * (n - 1) // 2} pairs)", "device_s": dev,
                     "host_oracle_s": time.perf_counter() - t0})
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "reps": args.reps, "rows": rows}
    for r in rows:
        print(f"{r['case']:<40} device {r['device_s'] * 1e3:9.2f} ms   host oracle {r['host_oracle_s'] * 1e3:10.1f} ms")
    print(json.dumps(info))


if __name__ == "__main__":
    main()
