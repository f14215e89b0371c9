"""Multi-view tracks and the COLMAP export (OmniVGGT.tracks: libovg ovg_match_* then ovg_tracks_*; colmap.write_colmap).

Workloads: 8 and 24 seeded surface-like 518^2 views at conf_percent=50, with all pairs and with the pairs of
compute_ranking(k=8) over a camera path.  Device: CUDA events over repeated calls after a warm-up, the matches (index and
query) and the assignment (assign, the one host read, gather) timed apart, and the whole call.  Host: write_colmap's time
and file sizes (binary, images=False), and the numpy oracle's track assembly from the same matches.  The device result is
checked equal to the oracle's.        python tools/tracks_bench.py [--reps 5] [--out DIR]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from match_bench import power_limit, scene, timed  # noqa: E402
from oracle import tracks_oracle as TO  # noqa: E402


def ranking_pairs(S, k=8):
    from omnivggt_official_b200.geometry import compute_ranking
    s = torch.linspace(0, 2, S, dtype=torch.float64)
    ext = torch.eye(4, dtype=torch.float64)[None].repeat(S, 1, 1)
    ext[:, :3, 3] = torch.stack([s.cos(), s.sin(), 0.1 * s], 1)
    ranking, _ = compute_ranking(ext.cuda(), k=k)
    return [(i, int(r)) for i, row in enumerate(ranking.cpu().tolist()) for r in row if r != i]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="write the result JSON here too")
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT, ops
    from omnivggt_official_b200.colmap import write_colmap
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cpus": os.cpu_count(), "rows": []}
    print(json.dumps({k: res[k] for k in ("gpu", "power_limit", "host_cpus")}), flush=True)
    for S in (8, 24):
        pred = scene(S)
        pred["images"] = torch.rand(1, S, 3, 518, 518, device="cuda", generator=torch.Generator(device="cuda").manual_seed(S))
        pred["intrinsic"] = torch.tensor([[466.2, 0, 259], [0, 466.2, 259], [0, 0, 1]], device="cuda").repeat(1, S, 1, 1)
        for label, pairs in (("all pairs", None), ("ranking k=8", ranking_pairs(S))):
            norm = TO.normalize_pairs(pairs, S).astype(np.int32)
            _, _, points, mask, _, _ = OmniVGGT._kept_views(pred, "depth", 50.0, 1e-5, None, 0, False)
            pair_off = np.searchsorted(norm[:, 0], np.arange(S + 1)).astype(np.int32)
            pairs_dev = torch.from_numpy(norm).cuda()
            off_dev = torch.from_numpy(pair_off).cuda()
            ext, intr = pred["extrinsic"][0].contiguous(), pred["intrinsic"][0].contiguous()
            images = pred["images"][0].contiguous()
            match_ms, mt = timed(lambda: ops.Matcher(points.view(S, -1, 3), mask.view(S, -1), pairs_dev), args.reps)

            def assign():
                tr = ops.Tracker(mt, off_dev, 2)
                n, m, _ = tr.counts()
                return tr.gather(images, ext, intr, 518, n, m)
            assign_ms, _ = timed(assign, args.reps)
            call_ms, out = timed(lambda: OmniVGGT.tracks(pred, pairs), args.reps)
            n, m = len(out["points"]), len(out["view"])
            # the oracle's assembly from the device's matches (test_tracks pins those to the cKDTree oracle)
            keep = mask.bool().view(S, 518, 518).cpu().numpy()
            rank = np.cumsum(keep.reshape(S, -1), 1) - 1
            matches = {}
            for (i, j), o in zip(norm.tolist(), OmniVGGT.matches(pred, [tuple(p) for p in norm.tolist()])):
                xi, xj = o["xy_i"].cpu().numpy(), o["xy_j"].cpu().numpy()
                matches[(i, j)] = (rank[i][xi[:, 1] * 518 + xi[:, 0]], rank[j][xj[:, 1] * 518 + xj[:, 0]])
            t = time.perf_counter()
            want = TO.scene_tracks(points.view(S, 518, 518, 3).cpu().numpy(), keep, images.cpu().numpy(), ext.cpu().numpy(),
                                   intr.cpu().numpy(), norm, 2, matches=matches)
            oracle_s = time.perf_counter() - t
            equal = all(np.array_equal(out[k].cpu().numpy(), want[k]) for k in want)
            with tempfile.TemporaryDirectory() as d:
                t = time.perf_counter()
                folder = write_colmap(d, pred, out, images=False)
                write_s = time.perf_counter() - t
                sizes = {f: os.path.getsize(os.path.join(folder, f)) for f in sorted(os.listdir(folder))}
            row = {"views": S, "pairs": label, "P": len(norm), "tracks": n, "observations": m,
                   "mean_track_length": round(m / max(n, 1), 3), "device_ms_matches": round(match_ms, 3),
                   "device_ms_tracks": round(assign_ms, 3), "device_ms_call": round(call_ms, 3),
                   "write_colmap_s": round(write_s, 3), "bytes": sizes, "oracle_assembly_s": round(oracle_s, 3),
                   "equal_to_oracle": equal}
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
            del mt, out
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "tracks_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
