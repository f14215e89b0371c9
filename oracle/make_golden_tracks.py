"""tests/golden/colmap.json: what the UNMODIFIED reference mat_to_quat (omnivggt/utils/rotation.py:47-109) returns in fp64 on
seeded rotations (build container only; TEST INFRASTRUCTURE).
python oracle/make_golden_tracks.py

rotation.py is loaded by file path; the reference tree is not touched.  The rotations hit each of the four argmax branches
(trace-dominant, and each axis-dominant, i.e. turns near 180 degrees about x, y and z), exact 180-degree turns, exact
90-degree turns about each axis (two branches tie), the identity and uniform random rotations.  The file holds each matrix
and the reference's scalar-last quaternion, as JSON floats (exact round trip)."""
from __future__ import annotations

import importlib.util
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
REFERENCE_ROTATION = "/root/reference/omnivggt/utils/rotation.py"


def rotations_of(q: np.ndarray) -> np.ndarray:
    """Rotation matrices [n, 3, 3] fp64 of quaternions q [n, 4] (w, x, y, z), normalised."""
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def make_rotations() -> np.ndarray:
    rng = np.random.default_rng(11)
    qs = [np.array([[1.0, 0.0, 0.0, 0.0]])]                                       # identity
    qs.append(np.array([[0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]]))   # exact 180-degree turns
    for axis in range(4):                                                           # each argmax branch, dominant component
        q = rng.standard_normal((6, 4)) * 0.2
        q[:, axis] = 1.0 + rng.random(6)
        qs.append(q)
    near = rng.standard_normal((6, 4)) * 1e-4                                       # within a few 1e-4 rad of 180 degrees
    near[np.arange(6), 1 + np.arange(6) % 3] = 1.0
    qs.append(near)
    qs.append(rng.standard_normal((12, 4)))                                         # uniform rotations
    R = rotations_of(np.concatenate(qs))
    R[0] = np.eye(3)
    turns = np.array([[[1, 0, 0], [0, 0, -1], [0, 1, 0]], [[0, 0, 1], [0, 1, 0], [-1, 0, 0]], [[0, -1, 0], [1, 0, 0], [0, 0, 1]]])
    return np.concatenate([R, turns.astype(np.float64)])                            # 90-degree turns: two branches tie


def main():
    import torch
    spec = importlib.util.spec_from_file_location("reference_rotation", REFERENCE_ROTATION)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    R = make_rotations()
    with torch.no_grad():
        q = mod.mat_to_quat(torch.from_numpy(R)).numpy()
    branches = np.argmax(np.stack([1 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2], 1 + R[:, 0, 0] - R[:, 1, 1] - R[:, 2, 2],
                                   1 - R[:, 0, 0] + R[:, 1, 1] - R[:, 2, 2], 1 - R[:, 0, 0] - R[:, 1, 1] + R[:, 2, 2]], 1), 1)
    assert set(branches.tolist()) == {0, 1, 2, 3}
    out = {"rotations": R.tolist(), "mat_to_quat_xyzw": q.tolist(), "_versions": {"torch": torch.__version__}}
    with open(os.path.join(GOLDEN, "colmap.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(len(R), "rotations, branches", np.bincount(branches).tolist())


if __name__ == "__main__":
    main()
