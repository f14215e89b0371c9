"""Point cloud on the device (OmniVGGT.point_cloud: libovg kernels) against the reference's host numpy path on seeded
predictions of 8 x 518^2 and 24 x 518^2.

Device: CUDA events around whole point_cloud calls (confidence select + mask, count, the one host read of the kept count,
gather, centre, scale) after a warm-up.  Host: the device-to-host copy of the per-pixel inputs it needs (world points,
confidence, images, cameras), then the GLB export's numpy steps (visual_util.py:190-236) and the viewer's
(inference.py:96-151), timed with perf_counter.        python tools/cloud_bench.py [--reps 20]"""
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
from oracle import pointcloud_oracle as PC  # noqa: E402


def inputs(S, H=518, W=518, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    world = torch.randn(S, H, W, 3, device="cuda", generator=g) * 3.0
    conf = 1.0 + torch.rand(S, H, W, device="cuda", generator=g).pow(3) * 8.0
    images = torch.rand(S, 3, H, W, device="cuda", generator=g)
    ext = torch.eye(4, device="cuda")[:3].repeat(S, 1, 1)
    return {"world_points_from_depth": world, "depth_conf": conf, "images": images, "extrinsic": ext}


def host_glb(world, conf, images, ext):
    """visual_util.py:196-236 on the host."""
    PC.point_cloud(world, conf, images, ext, 50.0, 1e-5, None, True, True)


def host_viewer(world, conf, images):
    """inference.py:98-143 on the host: flatten, colours, recentre on the mean, percentile mask, compaction."""
    pts = world.reshape(-1, 3)
    cols = PC.colors_u8(images)
    c = conf.reshape(-1)
    centered = pts - np.mean(pts, axis=0)
    thr = np.percentile(c, 50.0)
    keep = (c >= thr) & (c > 0.1) & PC.background_mask(cols, True, True)
    return centered[keep], cols[keep]


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3)
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cpus": os.cpu_count(), "sizes": []}
    for S in (8, 24):
        pred = inputs(S)
        kw = dict(conf_percent=50.0, mask_black_bg=True, mask_white_bg=True)
        for _ in range(3):
            OmniVGGT.point_cloud(pred, **kw)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.reps):
            cloud = OmniVGGT.point_cloud(pred, **kw)
        t1.record()
        torch.cuda.synchronize()
        dev_ms = t0.elapsed_time(t1) / args.reps
        d2h, glb, view = [], [], []
        for _ in range(args.host_reps):
            torch.cuda.synchronize()
            a = time.perf_counter()
            host = {k: v.cpu().numpy() for k, v in pred.items()}
            b = time.perf_counter()
            host_glb(host["world_points_from_depth"], host["depth_conf"], host["images"], host["extrinsic"])
            c = time.perf_counter()
            host_viewer(host["world_points_from_depth"], host["depth_conf"], host["images"])
            e = time.perf_counter()
            d2h.append(b - a), glb.append(c - b), view.append(e - c)
        row = {"views": S, "pixels": S * 518 * 518, "kept": int(cloud["points"].shape[0]), "device_ms": round(dev_ms, 3),
               "host_d2h_ms": round(1e3 * min(d2h), 2), "host_glb_ms": round(1e3 * min(glb), 1),
               "host_viewer_ms": round(1e3 * min(view), 1)}
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
