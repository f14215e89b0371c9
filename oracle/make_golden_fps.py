"""tests/golden/fps.json: what the UNMODIFIED reference farthest_point_sample (omnivggt/utils/po_utils/misc.py:114-148) returns
on a seeded case matrix (build container only; TEST INFRASTRUCTURE).
python oracle/make_golden_fps.py

misc.py is loaded by file path with its one unavailable import (prettytable, used only by count_parameters) stubbed; the
reference tree is not touched.  Per case: the input and output shapes and the SHA-256 of the int64 indices.  Cases with
deterministic=False draw the start from torch's default CPU generator after torch.manual_seed(seed)."""
from __future__ import annotations

import hashlib
import importlib.util
import json
import os
import sys
from unittest.mock import MagicMock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
REFERENCE_MISC = "/root/reference/omnivggt/utils/po_utils/misc.py"


def make_cases():
    """name -> dict(xyz [B, N, 3] float32 or float64, npoint, include_ends, deterministic, seed)."""
    from oracle.make_golden_matches import surface_views
    rng = np.random.default_rng(21)
    c = {}

    def case(name, xyz, npoint, include_ends=False, deterministic=True, seed=None):
        c[name] = dict(xyz=xyz, npoint=npoint, include_ends=include_ends, deterministic=deterministic, seed=seed)

    case("gaussian", rng.standard_normal((1, 4000, 3)).astype(np.float32), 256)
    case("b2", rng.standard_normal((2, 3000, 3)).astype(np.float32), 200)
    case("include_ends", rng.standard_normal((2, 2500, 3)).astype(np.float32), 128, include_ends=True)
    case("n1", rng.standard_normal((1, 1, 3)).astype(np.float32), 1)
    case("n1_include_ends", rng.standard_normal((2, 1, 3)).astype(np.float32), 1, include_ends=True)
    case("npoint_eq_n", rng.standard_normal((2, 300, 3)).astype(np.float32), 300)
    case("npoint_eq_n_include_ends", rng.standard_normal((1, 77, 3)).astype(np.float32), 77, include_ends=True)
    case("lattice_duplicates", rng.integers(0, 4, (1, 5000, 3)).astype(np.float32), 100)   # 64 positions: ties after 64
    case("all_equal", np.full((1, 500, 3), 0.75, np.float32), 20)
    sv = surface_views(S=2, H=48, W=64)
    case("surface", sv.reshape(1, -1, 3), 256)
    case("surface_views_b2", sv.reshape(2, -1, 3), 128)
    nf = rng.standard_normal((2, 2000, 3)).astype(np.float32)
    nf[0, [5, 300, 1999], 0] = np.nan
    nf[0, [17, 800], 1] = np.inf
    nf[0, [40, 1200], 2] = -np.inf
    nf[1, 0, 1] = np.nan                                                                   # the first sample is NaN
    nf[1, 900] = np.inf
    case("nonfinite", nf, 64)
    far = (rng.random((1, 3000, 3)) * 2e6 - 1e6).astype(np.float32)                        # d2 up to ~1e13 > 1e10
    far[0, :1000] *= 1e-4
    case("beyond_1e10", far, 64)
    case("float64", rng.standard_normal((1, 2000, 3)) * (1 + 1e-9), 100)
    case("random_start_seed0", rng.standard_normal((2, 2000, 3)).astype(np.float32), 64, deterministic=False, seed=0)
    case("random_start_seed1", rng.standard_normal((3, 1500, 3)).astype(np.float32), 64, include_ends=False,
         deterministic=False, seed=1)
    return c


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def load_reference_misc():
    sys.modules.setdefault("prettytable", MagicMock())
    spec = importlib.util.spec_from_file_location("reference_po_utils_misc", REFERENCE_MISC)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import torch
    misc = load_reference_misc()
    out = {}
    for name, k in make_cases().items():
        if k["seed"] is not None:
            torch.manual_seed(k["seed"])
        idx = misc.farthest_point_sample(torch.from_numpy(k["xyz"]), k["npoint"], include_ends=k["include_ends"],
                                         deterministic=k["deterministic"]).numpy().astype(np.int64)
        out[name] = {"xyz_shape": list(k["xyz"].shape), "xyz_dtype": str(k["xyz"].dtype), "inds_shape": list(idx.shape),
                     "inds_sha256": sha(idx), "xyz_sha256": sha(k["xyz"])}
        print(name, k["xyz"].shape, idx.shape, idx[:, :6].tolist())
    out["_versions"] = {"torch": torch.__version__, "numpy": np.__version__}
    with open(os.path.join(GOLDEN, "fps.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
