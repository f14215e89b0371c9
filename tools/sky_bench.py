"""Sky segmentation on the device (libovg ovg_segment_sky through OmniVGGT.sky_mask) against the reference's host recipe
(viz.py:357-393 segment_sky: cv2 HSV and colour test, scipy binary opening, cv2 connected components), and the whole
OmniVGGT.point_cloud call with and without mask_sky=True.

Device: CUDA events around whole calls after a warm-up, median of --reps; sky_mask is followed by its device-to-host copy of
the masks (the host read a caller that wants them on the host pays), point_cloud includes its own host reads.
Host: the same four library calls per view on the same images, already on the host as uint8 HWC, timed with perf_counter;
"not measured" when cv2 is missing.  Every device mask is checked equal to the host one.
        python tools/sky_bench.py [--reps 10]"""
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


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def images_of(S, H, W, seed, cell):
    """fp32 [S, 3, H, W] on the device: sky-coloured blobs and bright clouds over textured ground."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo = torch.rand(S, 1, H // cell + 2, W // cell + 2, device="cuda", generator=g)
    field = torch.nn.functional.interpolate(lo, size=(H, W), mode="bilinear", align_corners=False)[:, 0]
    y = torch.arange(H, device="cuda", dtype=torch.float32)[:, None] / H
    sky = torch.stack([0.27 + 0.3 * y, 0.5 + 0.2 * y, 0.92 - 0.1 * y]).expand(3, H, W)
    img = torch.where((field > 0.5)[:, None], sky[None], torch.rand(S, 3, H, W, device="cuda", generator=g) * 0.38)
    return torch.where((field > 0.8)[:, None], torch.full_like(img, 0.88), img).contiguous()


def host_segment_sky(u8):
    """The reference's four stages, by the same library calls, on uint8 [H, W, 3]."""
    import cv2
    from scipy import ndimage
    hsv = cv2.cvtColor(u8, cv2.COLOR_BGR2HSV)
    mask = cv2.inRange(hsv, np.array([0, 0, 100]), np.array([30, 255, 255])).view(bool)
    mask |= (hsv[:, :, 1] < 10) & (hsv[:, :, 2] > 150)
    mask |= (hsv[:, :, 1] < 30) & (hsv[:, :, 2] > 180)
    mask |= (hsv[:, :, 1] < 50) & (hsv[:, :, 2] > 220)
    opened = ndimage.binary_opening(mask, structure=np.ones((5, 5), np.uint8))
    _, labels, stats, _ = cv2.connectedComponentsWithStats(opened.view(np.uint8), connectivity=8)
    sizes = stats[1:, cv2.CC_STAT_AREA]
    keep = [1 + k for k in np.argsort(sizes)[::-1] if sizes[k] > sizes.max() / 2]
    return np.isin(labels, keep)


def _events(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT
    try:
        import cv2  # noqa: F401
        have_cv2 = True
    except ImportError:
        have_cv2 = False
    rows = []
    for S, H, W, cell in ((8, 518, 518, 24), (24, 518, 518, 24), (4, 3024, 4032, 300)):
        images = images_of(S, H, W, S, cell)
        pred = {"images": images}
        dev_ms, sky = _events(lambda: OmniVGGT.sky_mask(pred).cpu(), args.reps)
        row = {"views": S, "H": H, "W": W, "device_sky_mask_ms": round(dev_ms, 3), "sky_fraction": round(sky.float().mean().item(), 3)}
        if have_cv2:
            u8 = (images * 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous().cpu().numpy()
            ts = []
            for _ in range(max(3, args.reps // 3)):
                a = time.perf_counter()
                host = np.stack([host_segment_sky(u8[f]) for f in range(S)])
                ts.append(1e3 * (time.perf_counter() - a))
            ts.sort()
            row["host_reference_ms"] = round(ts[len(ts) // 2], 3)
            row["equal"] = bool(np.array_equal(host, sky.numpy()))
        else:
            row["host_reference_ms"] = "not measured (no cv2)"
        if H == 518:
            g = torch.Generator(device="cuda").manual_seed(1)
            pred.update(world_points_from_depth=torch.randn(S, H, W, 3, device="cuda", generator=g),
                        depth_conf=1.0 + torch.rand(S, H, W, device="cuda", generator=g),
                        extrinsic=torch.eye(4, device="cuda")[:3].repeat(S, 1, 1))
            row["point_cloud_ms"] = round(_events(lambda: OmniVGGT.point_cloud(pred), args.reps)[0], 3)
            row["point_cloud_mask_sky_ms"] = round(_events(lambda: OmniVGGT.point_cloud(pred, mask_sky=True), args.reps)[0], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "cpus": os.cpu_count(),
                      "rows": rows}))


if __name__ == "__main__":
    main()
