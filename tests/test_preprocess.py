"""Input pipeline (SURVEY.md section 8f rank 4).  CPU: the oracle (Pillow / OpenCV calls as in the reference + the restated tap and
index tables) against the UNMODIFIED reference loader's outputs on the seeded synthetic folders (tests/golden/preprocess.json).
GPU: the libovg kernels against the oracle, bit for bit on images / depth / mask."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import preprocess_oracle as PO
from oracle.synth_folder import FOLDERS, make_folder
from ovg_support import sha256

GOLD = json.load(open(os.path.join(GOLDEN, "preprocess.json")))


def _read_folder(d):
    """Host-side decode of a synthetic folder -> (images, cameras, depths, transposed) as the loaders take them."""
    from PIL import Image
    from omnivggt_official_b200.preprocess import read_camera_txt
    imgs, cams, deps, tr = [], [], [], []
    for p in sorted(os.listdir(d["images"])):
        stem = os.path.splitext(p)[0]
        img = Image.open(os.path.join(d["images"], p))
        if img.mode == "RGBA":
            img = Image.alpha_composite(Image.new("RGBA", img.size, (255, 255, 255, 255)), img)
        imgs.append(np.asarray(img.convert("RGB")))
        cpath = os.path.join(d["cameras"], stem + ".txt")
        cams.append(read_camera_txt(cpath) if os.path.exists(cpath) else None)
        dep, t = None, False
        if os.path.exists(os.path.join(d["depths"], stem + ".npy")):
            dep = np.load(os.path.join(d["depths"], stem + ".npy")).astype(np.float32)
        if os.path.exists(os.path.join(d["depths"], stem + ".png")):
            dep, t = np.asarray(Image.open(os.path.join(d["depths"], stem + ".png"))).astype(np.float32), True
        deps.append(dep)
        tr.append(t)
    return imgs, cams, deps, tr


@pytest.mark.parametrize("name", sorted(FOLDERS))
def test_oracle_matches_reference_loader(name, tmp_path):
    import PIL
    if PIL.__version__ != GOLD["_versions"]["pillow"]:
        pytest.skip("fixture hashes are for the pinned Pillow build")
    g = GOLD[name]
    imgs, cams, deps, tr = _read_folder(make_folder(str(tmp_path), name, seed=0))
    deps = [d.T if t else d for d, t in zip(deps, tr)]          # the reference transposes PNG depth (visual_util.py:771)
    images, extr, intr, dep, mask, didx, cidx = PO.load_views(imgs, cams, deps)
    assert list(images.shape) == g["images_shape"] and didx == g["depth_indices"] and cidx == g["camera_indices"]
    assert sha256(images.astype(np.float32)) == g["images_f32_sha256"]
    assert sha256(dep.astype(np.float32)) == g["depth_sha256"] and sha256(mask.astype(np.float32)) == g["mask_sha256"]
    assert np.allclose(extr, np.array(g["extrinsics"]), atol=2e-6) and np.allclose(intr, np.array(g["intrinsics"]), rtol=1e-5, atol=1e-3)


def test_tap_and_index_tables_match_the_libraries():
    import cv2
    from PIL import Image
    rng = np.random.default_rng(1)
    for (h, w, nh, nw) in ((480, 640, 392, 518), (500, 300, 868, 518), (389, 517, 392, 518), (97, 90, 560, 518)):
        im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = np.asarray(Image.fromarray(im).resize((nw, nh), Image.Resampling.BICUBIC))
        assert np.array_equal(PO.pil_resize_u8(im, nw, nh), ref)
    for (s, d) in ((480, 392), (512, 518), (163, 518), (1000, 518)):
        ramp = np.arange(s, dtype=np.float32)[None].repeat(2, 0)
        assert np.array_equal(cv2.resize(ramp, (d, 2), interpolation=cv2.INTER_NEAREST)[0].astype(int), PO.cv2_nearest_index(s, d))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FOLDERS))
def test_gpu_pipeline_matches_oracle_bit_for_bit(name, tmp_path):
    from omnivggt_official_b200 import preprocess as PP
    d = make_folder(str(tmp_path), name, seed=0)
    out = PP.load_images_and_cameras(d["images"], d["cameras"], d["depths"])
    torch.cuda.synchronize()
    check_pipeline_against_oracle(name, d, out)


def check_pipeline_against_oracle(name, d, out):
    """load_images_and_cameras' tuple for the synthetic folder d (make_folder(..., name)) against the oracle loader, and the
    image and depth digests of the reference's loader when Pillow is the pinned build."""
    imgs, cams, deps, tr = _read_folder(d)
    ref = PO.load_views(imgs, cams, [x.T if t else x for x, t in zip(deps, tr)])
    assert out[5] == ref[5] and out[6] == ref[6]
    assert torch.equal(out[0].cpu(), torch.from_numpy(ref[0]))                      # images: bit-exact
    assert torch.equal(out[3].cpu(), torch.from_numpy(ref[3])) and torch.equal(out[4].cpu(), torch.from_numpy(ref[4]))
    assert np.allclose(out[1].cpu().numpy(), ref[1], atol=2e-6) and np.allclose(out[2].cpu().numpy(), ref[2], rtol=1e-6, atol=1e-4)
    if PIL_version_matches():
        g = GOLD[name]
        assert sha256(out[0].cpu().numpy()) == g["images_f32_sha256"] and sha256(out[3].cpu().numpy()) == g["depth_sha256"]


def PIL_version_matches():
    import PIL
    return PIL.__version__ == GOLD["_versions"]["pillow"]


@pytest.mark.gpu
def test_gpu_pipeline_feeds_the_model(tmp_path):
    """The tuple goes straight into OmniVGGT.forward (the contract of inference.py:334-356)."""
    from omnivggt_official_b200 import preprocess as PP
    from test_model_gpu import model
    d = make_folder(str(tmp_path), "wide", seed=0)
    images, extr, intr, dep, mask, didx, cidx = PP.load_images_and_cameras(d["images"], d["cameras"], d["depths"], target_size=56)
    m = model("mini_conv")
    out = m(images=images, extrinsics=extr, intrinsics=intr, depth=dep, mask=mask, depth_gt_index=didx, camera_gt_index=cidx)
    assert out["depth"].shape == (1, 3, images.shape[-2], 56, 1) and torch.isfinite(out["world_points"]).all()
