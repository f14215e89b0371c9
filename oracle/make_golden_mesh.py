"""tests/golden/mesh.safetensors: the triangle meshes the UNMODIFIED reference builds on the host -- omnivggt/viz.py:40-77
(pts3d_to_trimesh) and :80-89 (cat_meshes) -- on the point cloud's seeded predictions and keep masks, plus mask and shape
edge cases (build container only; TEST INFRASTRUCTURE).        python oracle/make_golden_mesh.py

Inputs: the predictions of make_cloud_inputs with the reference's fp32 depth points and cameras from
tests/golden/point_cloud.safetensors, under the keep mask of every GLB_CASES case; then CASES below, each a list of views
(colours, points, valid mask) fed to the reference functions as they are.  Each mesh is stored as its face count and the
SHA-256 of its vertex, face and face-colour bytes.  trimesh is not needed by these two functions: viz.py only prints its
warning when it is absent."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden_cloud import GLB_CASES, digest, make_cloud_inputs  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")


def cloud_inputs():
    """(world_points_from_depth [S,H,W,3], depth_conf, images [S,3,H,W], world_points, world_points_conf, extrinsic [S,3,4]) of
    the point-cloud golden, as numpy."""
    from safetensors.torch import load_file
    g = load_file(os.path.join(GOLDEN, "point_cloud.safetensors"))
    inp = make_cloud_inputs()
    return {"world_points_from_depth": g["world_points_from_depth"].numpy(), "extrinsic": g["extrinsic"].numpy(),
            **{k: inp[k][0].numpy() for k in ("images", "depth_conf", "world_points", "world_points_conf")}}


def glb_case_views(g, case):
    """The views (colours uint8 [H,W,3], points fp32 [H,W,3], keep bool [H,W]) of one GLB_CASES case, with numpy's threshold."""
    from oracle import mesh_oracle as MO
    src, pct, frame, black, white = case
    world, conf = ((g["world_points_from_depth"], g["depth_conf"]) if src == "depth"
                   else (g["world_points"], g["world_points_conf"]))
    images = g["images"]
    if frame is not None:
        world, conf, images = world[frame][None], conf[frame][None], images[frame][None]
    keep, cols, _ = MO.keep_mask(conf, images, pct, 1e-5, black, white)
    return [(cols[f], world[f], keep[f]) for f in range(len(world))]


def _views(shapes, seed, masks, dtype=np.uint8):
    rng = np.random.default_rng(seed)
    out = []
    for (H, W), m in zip(shapes, masks):
        img = (rng.integers(0, 256, (H, W, 3)).astype(dtype) if dtype == np.uint8
               else rng.random((H, W, 3)).astype(dtype))
        out.append((img, rng.standard_normal((H, W, 3)).astype(np.float32), m))
    return out


def make_cases():
    """name -> list of views (img [H,W,3], pts3d fp32 [H,W,3], valid bool [H,W] or None)."""
    y, x = np.mgrid[0:9, 0:11]
    checker = (y + x) % 2 == 0                                   # no quad keeps three corners: no face survives
    isolated = np.zeros((9, 11), bool)
    isolated[1::3, 1::3] = True                                  # single pixels
    quads = np.zeros((9, 11), bool)
    quads[1:3, 1:3] = True                                       # one kept quad
    quads[5:7, 6:8] = True
    quads[4, 1] = quads[5, 1] = quads[4, 2] = True               # one TL triangle alone
    quads[1, 9] = quads[2, 8] = quads[2, 9] = True               # one BR triangle alone
    rng = np.random.default_rng(11)
    return {
        "all_kept": _views([(9, 11), (9, 11)], 1, [np.ones((9, 11), bool), None]),
        "checkerboard": _views([(9, 11), (9, 11)], 2, [checker, ~checker]),
        "isolated_pixels": _views([(9, 11)], 3, [isolated]),
        "single_quads": _views([(9, 11), (9, 11)], 4, [quads, quads[::-1, ::-1].copy()]),
        "one_row": _views([(1, 13), (1, 13)], 5, [np.ones((1, 13), bool), None]),
        "one_column": _views([(13, 1)], 6, [np.ones((13, 1), bool)]),
        "one_pixel": _views([(1, 1)], 7, [None]),
        "two_by_two": _views([(2, 2), (2, 2), (2, 2)], 8, [np.ones((2, 2), bool), np.eye(2, dtype=bool), None]),
        "random_float32": _views([(17, 23), (17, 23)], 9, [rng.random((17, 23)) < 0.7, rng.random((17, 23)) < 0.9],
                                 np.float32),
    }


def main():
    from safetensors.torch import save_file
    from oracle import mesh_oracle as MO
    from oracle.make_golden_cloud import _install_stand_ins
    from oracle.ref_shims import import_reference
    _install_stand_ins()
    sys.modules.pop("trimesh", None)                              # absent, as on a machine without it
    import_reference()
    from omnivggt import viz

    def record(out, key, views):
        ms = [viz.pts3d_to_trimesh(img.copy(), pts.copy(), None if v is None else v.copy()) for img, pts, v in views]
        m = viz.cat_meshes(ms)
        o = MO.cat_meshes([MO.pts3d_to_trimesh(img, pts, v) for img, pts, v in views])
        for k in ("vertices", "face_colors", "faces"):
            assert m[k].dtype == o[k].dtype and np.array_equal(m[k], o[k]), (key, k)
            out[f"{key}_{k}_sha256"] = digest(m[k])
        out[f"{key}_count"] = torch.tensor(len(m["faces"]), dtype=torch.int64)
        print(key, "faces", len(m["faces"]), "of", sum(4 * (i.shape[0] - 1) * (i.shape[1] - 1) for i, _, _ in views))

    g = cloud_inputs()
    out = {}
    for i, case in enumerate(GLB_CASES):
        record(out, f"glb{i}", glb_case_views(g, case))
    for name, views in make_cases().items():
        record(out, name, views)
    save_file({k: v.contiguous() for k, v in out.items()}, os.path.join(GOLDEN, "mesh.safetensors"))


if __name__ == "__main__":
    main()
