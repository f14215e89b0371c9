"""tests/golden/ranking.{json,npz}: what the UNMODIFIED reference compute_ranking (omnivggt/datasets/utils/image_ranking.py:
118-140) returns on a seeded case matrix (build container only; TEST INFRASTRUCTURE).
python oracle/make_golden_ranking.py

image_ranking.py is loaded by file path; the reference tree is not touched.  A case with `chunk` runs compute_ranking with
the module's extrinsic_distance_batch pointed at its own extrinsic_distance_batch_chunked(chunk_size=chunk), so the fp32
chunked formula is pinned at a small N.  Per case, ranking.json holds the parameters, the input's SHA-256 and the dtypes;
ranking.npz holds the dists (in the reference's dtype) and the ranking (as int16)."""
from __future__ import annotations

import functools
import hashlib
import importlib.util
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
REFERENCE_RANKING = "/root/reference/omnivggt/datasets/utils/image_ranking.py"


def rotations(q):
    """Rotation matrices of quaternions q [n, 4] (w, x, y, z), normalised."""
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def poses(rng, n, dtype=np.float64, rows=4, t_scale=3.0):
    """n random extrinsics [n, rows, 4]: uniform rotations, Gaussian translations, [0, 0, 0, 1] as the fourth row."""
    E = np.zeros((n, rows, 4))
    E[:, :3, :3] = rotations(rng.standard_normal((n, 4)))
    E[:, :3, 3] = rng.standard_normal((n, 3)) * t_scale
    if rows == 4:
        E[:, 3, 3] = 1.0
    return E.astype(dtype)


def trajectory(n, dtype):
    """A smooth video-like camera path: rotations a few thousandths of a radian apart, small steps along a curve."""
    s = np.arange(n) * 0.004
    half = 0.5 * np.stack([0.3 * np.sin(3 * s), s, 0.2 * np.cos(2 * s) - 0.2], 1)
    q = np.concatenate([np.ones((n, 1)), half], 1)
    E = np.zeros((n, 4, 4))
    E[:, :3, :3] = rotations(q)
    E[:, :3, 3] = np.stack([np.cos(s), np.sin(s), 0.05 * s], 1) * 2.0 + np.array([0.5, -0.2, 1.0])
    E[:, 3, 3] = 1.0
    return E.astype(dtype)


def make_cases():
    """name -> dict(E, lambda_t, normalize, batched, chunk)."""
    rng = np.random.default_rng(7)
    c = {}

    def case(name, E, lambda_t=1.0, normalize=True, batched=True, chunk=None):
        c[name] = dict(E=E, lambda_t=lambda_t, normalize=normalize, batched=batched, chunk=chunk)

    case("f32", poses(rng, 48, np.float32))
    case("f64", poses(rng, 64))
    case("f32_no_normalize", poses(rng, 40, np.float32), normalize=False)
    case("f64_no_normalize", poses(rng, 40), normalize=False)
    case("f64_lambda0", poses(rng, 32), lambda_t=0.0)
    case("f32_lambda2p5", poses(rng, 32, np.float32), lambda_t=2.5)
    case("f64_lambda_neg1", poses(rng, 32), lambda_t=-1.0)
    case("f32_lambda_neg1_no_normalize", poses(rng, 32, np.float32), lambda_t=-1.0, normalize=False)
    case("f64_rows3", poses(rng, 30, rows=3))
    case("loop_f32", poses(rng, 20, np.float32), batched=False)
    case("loop_f64", poses(rng, 20), batched=False)
    case("chunked_f64", poses(rng, 40), chunk=7)
    case("chunked_f32_lambda2p5", poses(rng, 33, np.float32), lambda_t=2.5, chunk=8)
    dup = poses(rng, 8)[rng.integers(0, 8, 40)]
    case("duplicates_f64", dup)
    case("duplicates_f32", dup.astype(np.float32), normalize=False)
    case("video_f32", trajectory(128, np.float32))
    case("video_f64", trajectory(64, np.float64))
    nanr = poses(rng, 16)
    nanr[5, 1, 2] = np.nan
    case("nan_rotation", nanr)
    nant = poses(rng, 12, np.float32)
    nant[3, 0, 3] = np.nan
    case("nan_translation_no_normalize", nant, normalize=False)
    zt = poses(rng, 10)
    zt[:, :3, 3] = 0.0
    case("zero_translations", zt)
    case("zero_translations_no_normalize", zt.copy(), normalize=False)
    case("n1", poses(rng, 1))
    case("n2_f32", poses(rng, 2, np.float32))
    return c


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def load_reference():
    spec = importlib.util.spec_from_file_location("reference_image_ranking", REFERENCE_RANKING)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_reference(mod, k):
    batch = mod.extrinsic_distance_batch
    if k["chunk"]:
        mod.extrinsic_distance_batch = functools.partial(mod.extrinsic_distance_batch_chunked, chunk_size=k["chunk"])
    try:
        with warnings.catch_warnings(), np.errstate(all="ignore"):
            warnings.simplefilter("ignore")
            return mod.compute_ranking(k["E"], lambda_t=k["lambda_t"], normalize=k["normalize"], batched=k["batched"])
    finally:
        mod.extrinsic_distance_batch = batch


def main():
    mod = load_reference()
    meta, arrays = {}, {}
    for name, k in make_cases().items():
        ranking, dists = run_reference(mod, k)
        meta[name] = {"E_shape": list(k["E"].shape), "E_dtype": str(k["E"].dtype), "E_sha256": sha(k["E"]),
                      "lambda_t": k["lambda_t"], "normalize": k["normalize"], "batched": k["batched"], "chunk": k["chunk"],
                      "dists_dtype": str(dists.dtype), "ranking_dtype": str(ranking.dtype)}
        arrays[f"{name}.dists"] = dists
        arrays[f"{name}.ranking"] = ranking.astype(np.int16)
        print(name, k["E"].shape, dists.dtype, ranking[0, :6].tolist())
    meta["_versions"] = {"numpy": np.__version__}
    np.savez_compressed(os.path.join(GOLDEN, "ranking.npz"), **arrays)
    with open(os.path.join(GOLDEN, "ranking.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
