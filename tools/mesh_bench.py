"""Triangle mesh on the device (OmniVGGT.mesh: libovg kernels) against the reference's host numpy recipe (viz.py:40-89
pts3d_to_trimesh + cat_meshes, restated in oracle/mesh_oracle.py) on seeded 518^2 views with the top half of each view kept.

Device, per layout, wall time (perf_counter) of whole calls after a warm-up:
  reference  OmniVGGT.mesh(layout="reference"): confidence select + mask, count, the one host read, faces; synchronised.
  glb        OmniVGGT.mesh(layout="glb") and glb.write_mesh_glb to a temporary file (device-to-host copy, bounds, file).
Host: the numpy recipe on the same inputs, already on the host, timed with perf_counter.
        python tools/mesh_bench.py [--reps 10]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mesh_oracle as MO  # noqa: E402


def inputs(S, H=518, W=518, seed=0):
    """Predictions of one scene; the confidence of the top half of each view is above that of the bottom half, so
    conf_percent=50 keeps a contiguous half of every view."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    world = torch.randn(S, H, W, 3, device="cuda", generator=g)
    conf = 1.0 + torch.rand(S, H, W, device="cuda", generator=g)
    conf[:, :H // 2] += 2.0
    images = torch.rand(S, 3, H, W, device="cuda", generator=g)
    ext = torch.eye(4, device="cuda")[:3].repeat(S, 1, 1)
    return {"world_points_from_depth": world, "depth_conf": conf, "images": images, "extrinsic": ext}


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def _wall(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        a = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - a)
    ts.sort()
    return 1e3 * ts[len(ts) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-reps", type=int, default=3)
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.glb import write_mesh_glb
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cpus": os.cpu_count(), "sizes": []}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "mesh.glb")
        for S in (8, 24):
            pred = inputs(S)

            def ref():
                return OmniVGGT.mesh(pred, conf_percent=50.0)

            def glb():
                m = OmniVGGT.mesh(pred, conf_percent=50.0, layout="glb")
                write_mesh_glb(path, m)
                return m

            for fn in (ref, glb):
                fn()
            ref_ms, r = _wall(ref, args.reps)
            glb_ms, gm = _wall(glb, args.reps)
            size = os.path.getsize(path)
            host = {k: v.cpu().numpy() for k, v in pred.items()}
            hs = []
            for _ in range(args.host_reps):
                a = time.perf_counter()
                o = MO.mesh(host["world_points_from_depth"], host["depth_conf"], host["images"], host["extrinsic"], 50.0)
                hs.append(time.perf_counter() - a)
            assert np.array_equal(o["faces"], r["faces"].cpu().numpy())           # both arms build the same mesh
            row = {"views": S, "pixels": S * 518 * 518, "faces": int(r["faces"].shape[0]),
                   "glb_faces": int(gm["indices"].shape[0]), "glb_vertices": int(gm["positions"].shape[0]),
                   "glb_bytes": size, "device_reference_ms": round(ref_ms, 2), "device_glb_with_write_ms": round(glb_ms, 1),
                   "host_reference_ms": round(1e3 * min(hs), 1)}
            res["sizes"].append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
