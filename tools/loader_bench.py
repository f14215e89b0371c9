"""Quick-start loader (preprocess.preprocess_images, libovg) against the reference's host path (load_fn.py:12-146: Pillow
bicubic resize, ToTensor, crop / white padding) on mixed phone-sized captures: 8 and 24 views alternating 1920 x 1080 landscape
and 3024 x 4032 portrait JPEGs, in crop and pad mode.

Decoding (Pillow, RGBA on white -> RGB) is the same for both and is timed on its own.  Both arms start from the decoded uint8
arrays: the host arm is oracle/load_fn_oracle.py with Pillow's own resize; the device arm is preprocess_images including the
host-to-device copies and a final synchronise, timed with perf_counter after a warm-up.  The two outputs are checked equal.
        python tools/loader_bench.py [--reps 5] [--host-reps 2]"""
from __future__ import annotations

import argparse
import contextlib
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
from oracle import load_fn_oracle as LO  # noqa: E402

SIZES = ((1920, 1080), (3024, 4032))        # (width, height), alternating


def write_views(d, n, seed=0):
    """n seeded smooth JPEGs (a random 64 x 48 image upscaled), alternating the two sizes."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    paths = []
    for i in range(n):
        w, h = SIZES[i % 2]
        small = Image.fromarray(rng.integers(0, 256, (48, 64, 3), dtype=np.uint8))
        p = os.path.join(d, f"view-{i:03d}.jpg")
        small.resize((w, h), Image.Resampling.BILINEAR).save(p, quality=90)
        paths.append(p)
    return paths


def pillow_resize(im, new_w, new_h):
    from PIL import Image
    return np.asarray(Image.fromarray(im).resize((new_w, new_h), Image.Resampling.BICUBIC))


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def best_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a = time.perf_counter()
        r = fn()
        ts.append(time.perf_counter() - a)
    return round(1e3 * min(ts), 2), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=2)
    args = ap.parse_args()
    from omnivggt_official_b200 import preprocess as PP
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "host_cpus": os.cpu_count(), "rows": []}
    print(json.dumps({k: res[k] for k in ("gpu", "power_limit", "host_cpus")}), flush=True)
    for n in (8, 24):
        with tempfile.TemporaryDirectory() as d:
            paths = write_views(d, n)
            decode_ms, images = best_ms(lambda: [PP.decode_rgb(p) for p in sorted(paths)], args.host_reps)
        for mode in ("crop", "pad"):
            with contextlib.redirect_stdout(io.StringIO()):          # the mixed-shape warning of crop mode
                PP.preprocess_images(images, mode)                  # warm-up: tap tables, allocator
                dev_ms, out = best_ms(lambda: PP.preprocess_images(images, mode), args.reps)
                host_ms, ref = best_ms(lambda: LO.preprocess_images(images, mode, resize=pillow_resize), args.host_reps)
            row = {"views": n, "mode": mode, "shape": list(out.shape), "decode_ms": decode_ms, "host_ms": host_ms,
                   "device_ms": dev_ms, "equal": bool(torch.equal(out.cpu(), torch.from_numpy(ref)))}
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
