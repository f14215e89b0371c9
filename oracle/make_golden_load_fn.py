"""tests/golden/load_fn.json: SHA-256 (and a strided sample) of what the UNMODIFIED reference quick-start loader
(omnivggt/utils/load_fn.py:12-146 load_and_preprocess_images) returns for seeded PNG lists, in crop and pad mode
(build container only; TEST INFRASTRUCTURE).        python oracle/make_golden_load_fn.py

The function imports with torch, Pillow and torchvision alone, so no shim is installed.  Per case and mode the file stores the
output shape, the SHA-256 of the float32 output and of rint(x * 255) as uint8 (ToTensor's output is uint8 / 255), a strided
uint8 sample and the warning line the reference prints for mixed shapes; "_versions" holds the Pillow build the digests are for."""
from __future__ import annotations

import contextlib
import hashlib
import io
import json
import os
import sys
import tempfile
from typing import Dict, List

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.ref_shims import REFERENCE_ROOT  # noqa: E402
from oracle.synth_folder import _image  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")
MODES = ("crop", "pad")

# name -> files in the order they are passed: (file name, width, height, kind); kind "rgb", "rgba" (composited on white) or
# "L" (grayscale, converted to RGB)
CASES: Dict[str, list] = {
    "landscape": [("view-0.png", 640, 480, "rgb"), ("view-1.png", 640, 480, "rgb")],
    "portrait": [("view-0.png", 300, 500, "rgb"), ("view-1.png", 300, 500, "rgb")],        # crop mode crops 868 -> 518 rows
    "mixed": [("a-landscape.png", 640, 480, "rgb"), ("b-portrait.png", 300, 500, "rgb"), ("c-square.png", 400, 400, "rgb"),
              ("d-rgba.png", 500, 375, "rgba"), ("e-gray.png", 350, 450, "L"), ("f-upscaled.png", 100, 60, "rgb")],
    "width518": [("view-0.png", 518, 700, "rgb")],        # crop mode: Pillow skips the horizontal pass
    "exact": [("view-0.png", 518, 392, "rgb")],           # no resampling in either mode
    "single": [("view-0.png", 1024, 300, "rgb")],
    "unsorted": [("c.png", 300, 500, "rgb"), ("a.png", 640, 480, "rgb"), ("b.png", 480, 480, "rgba")],
}


def write_case(root: str, name: str, seed: int = 0) -> List[str]:
    """Write the PNG files of one case under root/name; returns their paths in the case's (unsorted) order."""
    from PIL import Image
    d = os.path.join(root, name)
    os.makedirs(d, exist_ok=True)
    paths = []
    for i, (fname, w, h, kind) in enumerate(CASES[name]):
        img = _image(np.random.default_rng(seed + 7 * i + len(name)), h, w, rgba=(kind == "rgba"))
        if kind == "L":
            img = img[..., 1]
        p = os.path.join(d, fname)
        Image.fromarray(img).save(p)
        paths.append(p)
    return paths


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def summarize(x: np.ndarray, warning) -> dict:
    u8 = np.rint(np.asarray(x, np.float64) * 255).astype(np.uint8)
    return {"shape": list(x.shape), "f32_sha256": digest(np.asarray(x, np.float32)), "u8_sha256": digest(u8),
            "samples": u8[:, :, ::97, ::89].tolist(), "warning": warning}


def main():
    sys.path.insert(0, REFERENCE_ROOT)
    from omnivggt.utils.load_fn import load_and_preprocess_images
    res = {}
    with tempfile.TemporaryDirectory() as root:
        for name in CASES:
            paths = write_case(root, name)
            res[name] = {}
            for mode in MODES:
                buf = io.StringIO()
                with contextlib.redirect_stdout(buf):
                    x = load_and_preprocess_images(list(paths), mode=mode).numpy()
                res[name][mode] = summarize(x, buf.getvalue().strip() or None)
                print(name, mode, list(x.shape), res[name][mode]["warning"])
    import PIL
    res["_versions"] = {"pillow": PIL.__version__}
    with open(os.path.join(GOLDEN, "load_fn.json"), "w") as f:
        json.dump(res, f, sort_keys=True, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
