"""tests/golden/sky.safetensors: the sky masks the UNMODIFIED reference computes on the host -- omnivggt/viz.py:357-393
(segment_sky) -- on seeded synthetic images, and the point clouds of predictions_to_glb(..., mask_sky=True)
(visual_util.py:140-236) with those masks as its mask files (build container only; TEST INFRASTRUCTURE).
        python oracle/make_golden_sky.py

segment_sky cases: make_cases below; each mask is stored as its sky-pixel count and the SHA-256 of np.packbits(mask).
GLB cases: the point-cloud golden's predictions (make_golden_mesh.cloud_inputs) with a sky painted into the images
(sky_cloud_inputs), under every GLB_CASES setting.  The reference reads one mask file per image name from
<target_dir>/sky_masks (uint8, 255 = non-sky); they are written as PNG (lossless) at H x W, so no resize happens.  The
reference's ONNX sky network is never reached: the working directory holds an empty skyseg.onnx (so nothing is downloaded),
every mask file exists (so no session is created), and download_file_from_url, onnxruntime.InferenceSession and requests are
replaced by functions that raise."""
from __future__ import annotations

import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle.make_golden_cloud import GLB_CASES, REC, digest  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(HERE), "tests", "golden")


def mask_digest(mask: np.ndarray) -> torch.Tensor:
    return digest(np.packbits(np.ascontiguousarray(mask, dtype=bool)))


def sky_rows(H: int, W: int, seed: int) -> np.ndarray:
    """A blue sky gradient as RGB uint8 [H, W, 3] (H <= 30 in OpenCV's hue once read as BGR), with a little noise."""
    rng = np.random.default_rng(seed)
    y = np.arange(H)[:, None] * np.ones((1, W))
    img = np.stack([70 + 2 * y, 130 + y, 235 - y], -1) + rng.integers(-3, 4, (H, W, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def ground(H: int, W: int, seed: int) -> np.ndarray:
    """Textured ground, every channel below 100: never sky-coloured."""
    return np.random.default_rng(seed).integers(0, 100, (H, W, 3)).astype(np.uint8)


def _paint(img, m, color):
    img[m] = np.array(color, np.uint8)
    return img


def make_cases():
    """name -> image [H, W, 3] (uint8, float32 or float64)."""
    c = {}
    H, W = 64, 96
    img = ground(H, W, 1)
    img[:28] = sky_rows(28, W, 2)
    c["gradient_over_ground"] = img

    img = ground(H, W, 3)
    img[:30] = sky_rows(30, W, 4)
    img[4:14, 10:40] = (228, 230, 236)                          # cloud: low saturation, bright
    img[16:24, 50:80] = (196, 198, 204)                         # grey cloud: S < 30, V > 180
    img[6:12, 60:70] = (240, 240, 240)
    c["clouds"] = img

    img = ground(H, W, 5)
    img[:18, :40] = sky_rows(18, 40, 6)                         # 720 px of sky
    img[30:64, 50:96] = (250, 250, 250)                         # 1564 px of white wall: the sky is dropped
    c["white_wall_wins"] = img
    img = ground(H, W, 7)
    img[:20, :60] = sky_rows(20, 60, 8)                         # 1200 px of sky
    img[34:58, 70:96] = (245, 246, 250)                         # 624 px of wall: both kept
    c["white_wall_competes"] = img

    img = sky_rows(40, 80, 9)
    for x0 in (15, 35, 55):                                     # three trunks, 1, 2 and 3 px wide, cut four equal sky parts
        img[:, x0:x0 + 1] = (40, 70, 30)
    img[:, 16:20] = (40, 70, 30)                                # widen to equal parts of 15 columns each
    img[:, 36:40] = (40, 70, 30)
    img[:, 56:60] = (40, 70, 30)
    img[:, 75:80] = (40, 70, 30)
    c["trees_equal_parts"] = img

    img = ground(40, 60, 10)
    s = sky_rows(40, 60, 11)
    m = np.zeros((40, 60), bool)
    m[2:9, 2:12] = True                                         # 7 x 10 = 70: the largest
    m[15:20, 2:9] = True                                        # 5 x 7 = 35 = 70 / 2: dropped
    m[25:31, 20:26] = True                                      # 6 x 6 = 36: kept
    img[m] = s[m]
    c["half_area_even"] = img
    img = ground(40, 60, 12)
    m = np.zeros((40, 60), bool)
    m[2:9, 2:11] = True                                         # 7 x 9 = 63: the largest, odd
    m[15:20, 2:8] = True                                        # 30: dropped
    m[15:20, 20:27] = True                                      # 35: kept
    m[25:30, 30:35] = True                                      # two 5 x 5 squares offset by (1, 1): 34, kept
    m[26:31, 31:36] = True
    img[m] = s[m]
    c["half_area_odd"] = img

    img = ground(48, 64, 13)
    img[30:48, 40:64] = sky_rows(18, 24, 14)                    # a block that survives
    img[5, :] = (120, 160, 240)                                 # 1 px line
    img[10:12, 5:60] = (120, 160, 240)                          # 2 px line
    img[:, 20] = (250, 250, 250)
    img[14:28, 30:32] = (250, 250, 250)
    img[20:24, 40:44] = (120, 160, 240)                         # 4 x 4 square: below the 5 x 5 box
    c["thin_structures"] = img

    img = sky_rows(50, 70, 15)
    img[8:42, 8:62] = ground(34, 54, 16)                        # a ring of sky touching every border
    c["sky_on_every_border"] = img

    c["all_sky"] = sky_rows(33, 45, 17)
    c["no_sky"] = ground(33, 45, 18)
    y, x = np.mgrid[0:32, 0:48]
    c["checkerboard"] = _paint(ground(32, 48, 19), (y + x) % 2 == 0, (120, 160, 240))

    rng = np.random.default_rng(20)
    from scipy import ndimage
    blobs = ndimage.uniform_filter(rng.random((72, 88)), 9) > 0.5
    img = ground(72, 88, 21)
    img[blobs] = sky_rows(72, 88, 22)[blobs]
    c["random_blobs"] = img

    for h, w in ((1, 9), (9, 1), (1, 1), (4, 4), (5, 5), (4, 9), (9, 4), (5, 9), (9, 5)):
        c[f"tiny_{h}x{w}"] = sky_rows(h, w, 23)

    base = c["clouds"].astype(np.float64) / 255.0
    rng = np.random.default_rng(24)
    wild = base + rng.uniform(-0.4, 0.4, base.shape) * (rng.random(base.shape) < 0.2)   # values outside [0, 1]
    c["float64_out_of_range"] = wild
    c["float32_out_of_range"] = wild.astype(np.float32)
    c["float32_gradient"] = (c["gradient_over_ground"].astype(np.float32) / np.float32(255))
    return c


def sky_cloud_inputs():
    """The point-cloud golden's predictions (numpy, one scene) with a sky painted into rows 0-11 of every view (away from the
    black and white patches of views 0 and 1) and a cloud in view 1."""
    from oracle.make_golden_mesh import cloud_inputs
    g = cloud_inputs()
    images = g["images"].copy()
    S, _, H, W = images.shape
    for f in range(S):
        x0 = 12 + 8 * f
        sky = sky_rows(12, W - x0, 30 + f).astype(np.float32) / np.float32(255)
        images[f, :, :12, x0:] = np.transpose(sky, (2, 0, 1))
    images[1, :, 2:7, 30:45] = np.float32(0.9)
    g["images"] = images
    return g


def main():
    import cv2
    from safetensors.torch import save_file
    from oracle import sky_oracle as SO
    from oracle.make_golden_cloud import _install_stand_ins
    from oracle.ref_shims import import_reference

    def refuse(*a, **k):
        raise RuntimeError("the sky network must not be reached")

    _install_stand_ins()
    requests = types.ModuleType("requests")
    requests.get = requests.post = requests.head = requests.request = requests.Session = refuse   # any request raises
    requests.exceptions = types.SimpleNamespace(RequestException=RuntimeError)
    sys.modules["requests"] = requests
    sys.modules["onnxruntime"].InferenceSession = refuse
    import_reference()
    from omnivggt import viz
    import visual_util as vu
    vu.download_file_from_url = refuse
    vu.requests = requests

    out = {}
    for name, img in make_cases().items():
        m = viz.segment_sky(img.copy()).numpy()
        assert m.dtype == bool and m.shape == img.shape[:2], name
        assert np.array_equal(m, SO.segment_sky(img)), name
        out[f"{name}_count"] = torch.tensor(int(m.sum()), dtype=torch.int64)
        out[f"{name}_sha256"] = mask_digest(m)
        print(name, img.shape, img.dtype, "sky", int(m.sum()))

    g = sky_cloud_inputs()
    S, _, H, W = g["images"].shape
    out["images_sha256"] = digest(g["images"])
    sky = np.stack([viz.segment_sky(np.ascontiguousarray(np.transpose(g["images"][f], (1, 2, 0)))).numpy() for f in range(S)])
    assert np.array_equal(sky, SO.sky_of_views(g["images"]))
    out["views_sky_sha256"] = mask_digest(sky)
    print("views sky", sky.reshape(S, -1).sum(1))
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "images"))
        os.makedirs(os.path.join(tmp, "sky_masks"))
        open(os.path.join(tmp, "skyseg.onnx"), "wb").close()
        for f in range(S):
            name = f"{f:03d}.png"
            cv2.imwrite(os.path.join(tmp, "images", name), np.zeros((H, W, 3), np.uint8))
            cv2.imwrite(os.path.join(tmp, "sky_masks", name), (255 * ~sky[f]).astype(np.uint8))
        os.chdir(tmp)
        try:
            for i, (src, pct, frame, black, white) in enumerate(GLB_CASES):
                REC.clear()
                p = {k: v.copy() for k, v in g.items()}
                if src != "depth":
                    p.pop("world_points_from_depth")
                vu.predictions_to_glb(p, conf_thres=pct, filter_by_frames="All" if frame is None else f"{frame}: view",
                                      mask_black_bg=black, mask_white_bg=white, show_cam=True, mask_sky=True, target_dir=tmp,
                                      prediction_mode="Predicted Depth" if src == "depth" else "Predicted Pointmap")
                world, conf = ((g["world_points_from_depth"], g["depth_conf"]) if src == "depth"
                               else (g["world_points"], g["world_points_conf"]))
                o = SO.point_cloud(world, conf, g["images"], g["extrinsic"], sky, pct, 1e-5, frame, black, white)
                if len(o["points"]):
                    assert np.array_equal(REC["points"], o["points"]) and np.array_equal(REC["colors"], o["colors"]), i
                out[f"glb{i}_count"] = torch.tensor(len(REC["points"]), dtype=torch.int64)
                out[f"glb{i}_points_sha256"] = digest(REC["points"])
                out[f"glb{i}_colors_sha256"] = digest(REC["colors"])
                c = SO.mask_conf(conf, sky)
                c = (c if frame is None else c[frame]).reshape(-1)
                out[f"glb{i}_thr"] = torch.tensor(float(0.0 if pct == 0.0 else np.percentile(c, pct)), dtype=torch.float64)
                print("glb", i, GLB_CASES[i], "kept", len(o["points"]))
        finally:
            os.chdir(cwd)
    save_file({k: v.contiguous() for k, v in out.items()}, os.path.join(GOLDEN, "sky.safetensors"))


if __name__ == "__main__":
    main()
