"""tests/golden/matches.json: what the UNMODIFIED reference find_reciprocal_matches (omnivggt/utils/geometry.py:435-451, two
cKDTree builds and queries) returns on a seeded case matrix (build container only; TEST INFRASTRUCTURE).
python oracle/make_golden_matches.py

Per case: the sizes, the match count, the SHA-256 of reciprocal_in_P2 (bool) and nn2_in_P1 (int64), the SHA-256 of cKDTree's
neighbour distances in both directions (fp64), and whether the case has exact ties (where cKDTree's choice of neighbour is
unspecified, so only its distances are pinned)."""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")


def surface_views(S=2, H=48, W=64, seed=3):
    """Point maps unprojected from a smooth synthetic depth with slightly different cameras: [S, H, W, 3] fp32."""
    rng = np.random.default_rng(seed)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    out = []
    for s in range(S):
        depth = 2.0 + 0.3 * np.sin(u / 9.0 + s) + 0.2 * np.cos(v / 7.0) + 0.01 * rng.standard_normal((H, W))
        f = 0.9 * W
        x = (u - W / 2 + 1.5 * s) * depth / f
        y = (v - H / 2) * depth / f
        a = 0.05 * s
        pts = np.stack([np.cos(a) * x + np.sin(a) * depth, y, -np.sin(a) * x + np.cos(a) * depth + 0.02 * s], -1)
        out.append(pts)
    return np.stack(out).astype(np.float32)


def make_cases():
    """name -> (P1, P2) fp32 [n, 3] / [m, 3]."""
    rng = np.random.default_rng(11)
    c = {}
    c["uniform"] = (rng.random((3000, 3)), rng.random((2500, 3)))
    centers = rng.standard_normal((6, 3)) * 5
    c["clustered"] = tuple(centers[rng.integers(0, 6, n)] + 0.05 * rng.standard_normal((n, 3)) for n in (2800, 3200))
    sv = surface_views()
    c["surface"] = (sv[0].reshape(-1, 3), sv[1].reshape(-1, 3))
    c["duplicates"] = (rng.integers(0, 6, (2000, 3)), rng.integers(0, 6, (1500, 3)))
    c["all_equal"] = (np.full((50, 3), 0.25), np.full((40, 3), -1.5))
    c["all_equal_same"] = (np.full((30, 3), 2.0), np.full((45, 3), 2.0))
    c["planar"] = (np.c_[rng.random((2000, 2)), np.zeros(2000)], np.c_[rng.random((1800, 2)), np.zeros(1800)])
    c["collinear"] = (np.c_[rng.random(1500), np.zeros((1500, 2))], np.c_[rng.random(1700), np.zeros((1700, 2))])
    far1, far2 = rng.random((2500, 3)), rng.random((2200, 3))
    far1[17] = (1e6, -3e5, 2e6)
    c["far_outlier"] = (far1, far2)
    c["one_vs_10k"] = (rng.random((1, 3)), rng.random((10000, 3)))
    c["10k_vs_one"] = (rng.random((10000, 3)), rng.random((1, 3)))
    from safetensors.numpy import load_file
    pc = load_file(os.path.join(GOLDEN, "point_cloud.safetensors"))["world_points_from_depth"]   # [3, 42, 70, 3]
    c["point_cloud_01"] = (pc[0].reshape(-1, 3), pc[1].reshape(-1, 3))
    c["point_cloud_21"] = (pc[2].reshape(-1, 3), pc[1].reshape(-1, 3))
    return {k: (np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)) for k, (a, b) in c.items()}


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    from scipy.spatial import cKDTree
    from oracle import matches_oracle as MO
    from oracle.ref_shims import import_reference
    import_reference()
    from omnivggt.utils import geometry
    out = {}
    for name, (P1, P2) in make_cases().items():
        rec, nn2, count = geometry.find_reciprocal_matches(P1, P2)
        d1, _ = cKDTree(P2).query(P1)
        d2, _ = cKDTree(P1).query(P2)
        out[name] = {"n": len(P1), "m": len(P2), "count": int(count), "reciprocal_sha256": sha(np.asarray(rec, bool)),
                     "nn2_in_P1_sha256": sha(np.asarray(nn2, np.int64)), "dist1_sha256": sha(d1.astype(np.float64)),
                     "dist2_sha256": sha(d2.astype(np.float64)),
                     "has_ties": MO.has_ties(P1, P2) or MO.has_ties(P2, P1)}
        print(name, out[name]["n"], out[name]["m"], out[name]["count"], "ties" if out[name]["has_ties"] else "")
    import scipy
    out["_versions"] = {"scipy": scipy.__version__, "numpy": np.__version__}
    with open(os.path.join(GOLDEN, "matches.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
