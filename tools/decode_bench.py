"""Device JPEG decoding (preprocess.decode_images, csrc/jpeg.cuh) against Pillow, on camera-like octave-noise JPEGs
(oracle/jpeg_oracle.octave_noise: 2-5 bits per pixel, like camera files; smooth upscaled images would flatter the Huffman stage).

Sets: 8 and 24 views alternating 1920 x 1080 / 3024 x 4032 at 4:2:0 quality 90 (phone captures), and 4 and 16 views of
6048 x 4032 at 4:2:2 quality 95 (camera captures).  Per set: compressed size and bits per pixel; serial Pillow decode; decode_images
split into plan + unstuff (host), the host-to-device copy and the kernels (CUDA events, sync rounds included), and end to end with
a final synchronise; the most sync rounds; the folder-to-tensors loader with host decoding (before) and with decode_images
(after) -- load_images_and_cameras for the camera sets, load_and_preprocess_images (crop) for the mixed-orientation sets, whose
views do not resize to one height; and whether every output equals Pillow's.  Prints the GPU name, power limit and CPU count.
        python tools/decode_bench.py [--reps 3]"""
from __future__ import annotations

import argparse
import contextlib
import ctypes
import io
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
from oracle import jpeg_oracle as J  # noqa: E402

SETS = [("phone 8", 8, ((1920, 1080), (3024, 4032)), dict(quality=90, subsampling=2)),
        ("phone 24", 24, ((1920, 1080), (3024, 4032)), dict(quality=90, subsampling=2)),
        ("camera 4", 4, ((6048, 4032),), dict(quality=95, subsampling=1)),
        ("camera 16", 16, ((6048, 4032),), dict(quality=95, subsampling=1))]


def write_set(d, n, sizes, kw):
    """n files; four distinct images per size, reused cyclically (generating 6048 x 4032 noise is slow on the host)."""
    cache, paths = {}, []
    for i in range(n):
        w, h = sizes[i % len(sizes)]
        key = (w, h, (i // len(sizes)) % 4)
        if key not in cache:
            cache[key] = J.encode(J.octave_noise(w, h, seed=hash(key) & 0xFFFF), **kw)
        p = os.path.join(d, f"view-{i:03d}.jpg")
        with open(p, "wb") as f:
            f.write(cache[key])
        paths.append(p)
    return paths


def timed(fn, reps):
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t)
    return best * 1e3, r


def phases(paths):
    """decode_images' steps with a clock / CUDA events around each: (plan ms, copy ms, kernels ms, rounds)."""
    from omnivggt_official_b200 import _lib as L
    t = time.perf_counter()
    plan = L.JpegPlan([open(p, "rb").read() for p in paths])
    staging = torch.empty(plan.stream_bytes, dtype=torch.uint8, pin_memory=True)
    plan.fill_stream(staging.data_ptr())
    t_plan = (time.perf_counter() - t) * 1e3
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device="cuda")
    st = torch.zeros(len(paths), dtype=torch.int32, device="cuda")
    outs = [torch.empty(f[1], f[2], 3, dtype=torch.uint8, device="cuda") for f in plan.files]
    ptrs = (ctypes.c_void_p * len(paths))(*[o.data_ptr() for o in outs])
    ev[0].record()
    stream = staging.to("cuda", non_blocking=True)
    ev[1].record()
    L.check(L.lib().ovg_jpeg_decode(plan.handle, stream.data_ptr(), ptrs, st.data_ptr(), ws.data_ptr(), plan.workspace_bytes,
                                    L.stream()))
    ev[2].record()
    torch.cuda.synchronize()
    assert not st.any()
    return t_plan, ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), plan.rounds()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from omnivggt_official_b200 import preprocess as PP
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    print(f"GPU: {gpu}; host CPUs: {os.cpu_count()}")
    rows = []
    for name, n, sizes, kw in SETS:
        with tempfile.TemporaryDirectory() as d:
            paths = write_set(d, n, sizes, kw)
            nbytes = sum(os.path.getsize(p) for p in paths)
            pix = sum(w * h for w, h in (sizes[i % len(sizes)] for i in range(n)))
            t_pil, host = timed(lambda: [PP.decode_rgb(p) for p in paths], 1)
            PP.decode_images(paths)                                       # warm-up
            t_dev, dev = timed(lambda: PP.decode_images(paths), args.reps)
            equal = all(np.array_equal(a.cpu().numpy(), b) for a, b in zip(dev, host))
            ph = [phases(paths) for _ in range(args.reps)]
            best = min(ph, key=lambda r: r[0] + r[1] + r[2])
            if len(sizes) == 1:
                loader = "load_images_and_cameras"
                before = lambda: PP.preprocess_views([PP.decode_rgb(p) for p in paths])             # noqa: E731
                after = lambda: PP.load_images_and_cameras(d)                                     # noqa: E731
            else:
                loader = "load_and_preprocess_images"
                before = lambda: PP.preprocess_images([PP.decode_rgb(p) for p in paths])           # noqa: E731
                after = lambda: PP.load_and_preprocess_images(paths)                              # noqa: E731
            with contextlib.redirect_stdout(io.StringIO()):
                after()
                t_before, rb = timed(before, 1)
                t_after, ra = timed(after, args.reps)
            same = torch.equal(rb[0] if isinstance(rb, tuple) else rb, ra[0] if isinstance(ra, tuple) else ra)
            row = dict(set=name, views=n, MB=round(nbytes / 1e6, 1), bits_per_pixel=round(8 * nbytes / pix, 2),
                       pillow_ms=round(t_pil, 1), decode_images_ms=round(t_dev, 1), plan_unstuff_ms=round(best[0], 1),
                       h2d_ms=round(best[1], 2), kernels_ms=round(best[2], 2), max_rounds=max(r[3] for r in ph),
                       loader=loader, loader_before_ms=round(t_before, 1), loader_after_ms=round(t_after, 1),
                       equal=bool(equal and same))
            print(json.dumps(row), flush=True)
            rows.append(row)
    print("| set | views | MB | bits/px | Pillow | decode_images | plan + unstuff | H2D | kernels | max rounds | loader "
          "before → after | equal |")
    for r in rows:
        print(f"| {r['set']} | {r['views']} | {r['MB']} | {r['bits_per_pixel']} | {r['pillow_ms']} ms | "
              f"{r['decode_images_ms']} ms | {r['plan_unstuff_ms']} ms | {r['h2d_ms']} ms | {r['kernels_ms']} ms | "
              f"{r['max_rounds']} | {r['loader_before_ms']} → {r['loader_after_ms']} ms | {r['equal']} |")


if __name__ == "__main__":
    main()
