"""Bundle adjustment of tracks (OmniVGGT.bundle_adjust: libovg ovg_bundle_adjust).

Workloads: tools/tracks_bench.py's seeded surface-like 518^2 views, 8 views with all pairs and 24 views with the pairs of
compute_ranking(k=8), the cameras handed to tracks() perturbed by a seeded 0.01 rad rotation, 1 % of the translation and 2 %
of the focal length.  Device: CUDA events over repeated calls after a warm-up, per call and per LM step.  Reported: steps,
accepted steps and PCG iterations, initial and final cost, mean track error before and after, the workspace bytes, and the
numpy oracle's host time on the same problem (at most --oracle-iterations steps, scaled per step).
        python tools/ba_bench.py [--reps 3] [--out FILE]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from match_bench import power_limit, scene, timed  # noqa: E402
from tracks_bench import ranking_pairs  # noqa: E402
from oracle import ba_oracle as BO  # noqa: E402


def surface_cameras(S, H, W):
    """The world-to-camera cameras oracle.make_golden_matches.surface_views unprojects through (f = 0.9 W, principal point
    (W/2 - 1.5 s, H/2), a rotation of 0.05 s about y and a 0.02 s shift in z), perturbed: rotation 0.01 rad, translation 1 %,
    focal 2 %, seeded."""
    rng = np.random.default_rng(S)
    ext, intr = np.zeros((S, 3, 4)), np.zeros((S, 3, 3))
    for s in range(S):
        a = 0.05 * s
        rcw = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        ext[s] = np.c_[BO.exp_so3(0.01 * rng.standard_normal(3) / np.sqrt(3)) @ rcw.T,
                       -rcw.T @ np.array([0, 0, 0.02 * s]) * (1 + 0.01 * rng.standard_normal(3))]
        f = 0.9 * W * (1 + 0.02 * rng.standard_normal())
        intr[s] = [[f, 0, W / 2 - 1.5 * s], [0, f, H / 2], [0, 0, 1]]
    return torch.from_numpy(ext).float().cuda(), torch.from_numpy(intr).float().cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iterations", type=int, default=100)
    ap.add_argument("--oracle-iterations", type=int, default=3)
    ap.add_argument("--out", default=None, help="write the result JSON here too")
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT, _lib
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cpus": os.cpu_count(), "rows": []}
    print(json.dumps({k: res[k] for k in ("gpu", "power_limit", "host_cpus")}), flush=True)
    for S, label, pairs in ((8, "all pairs", None), (24, "ranking k=8", "ranking")):
        pred = scene(S)
        pred["extrinsic"], pred["intrinsic"] = (t[None] for t in surface_cameras(S, 518, 518))
        tr = OmniVGGT.tracks(pred, ranking_pairs(S) if pairs else None)
        n, m = len(tr["points"]), len(tr["view"])
        call_ms, out = timed(lambda: OmniVGGT.bundle_adjust(tr, iterations=args.iterations), args.reps)
        ba = {k: v.cpu().tolist() for k, v in out["ba"].items()}
        fin = torch.isfinite(tr["error"])
        t = time.perf_counter()
        host = [x.cpu().numpy() for x in (tr["points"], tr["offsets"], tr["view"], tr["xy"].double() + 0.5, tr["extrinsic"],
                                          tr["intrinsic"])]
        o = BO.bundle_adjust(*host, iterations=args.oracle_iterations)
        oracle_s = time.perf_counter() - t
        row = {"views": S, "pairs": label, "tracks": n, "observations": m,
               "workspace_bytes": _lib.load().ovg_ba_workspace_bytes(S, n, m),
               "device_ms_per_call": round(call_ms, 2), "device_ms_per_step": round(call_ms / max(ba["steps"], 1), 3),
               "steps": ba["steps"], "accepted": ba["accepted"], "pcg_iterations": ba["pcg_iterations"], "status": ba["status"],
               "cost": ba["cost"], "mean_error_px": [float(tr["error"][fin].mean()), float(out["error"][fin].mean())],
               "oracle_s_per_step": round(oracle_s / max(o["steps"], 1), 2), "oracle_steps": o["steps"]}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
