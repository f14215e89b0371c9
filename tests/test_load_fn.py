"""Quick-start loader (reference omnivggt/utils/load_fn.py:12-146, load_and_preprocess_images): crop and pad mode, mixed sizes
padded with white.  CPU: the numpy oracle against the UNMODIFIED reference's outputs on seeded PNG lists (tests/golden/
load_fn.json), the package's geometry against where the oracle places each image, the errors, and a dry run of the library calls.
GPU: libovg against the oracle and the golden, bit for bit; ovg_preprocess_image_canvas on its own; the output feeding the model."""
import hashlib
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import load_fn_oracle as LO
from oracle import preprocess_oracle as PO
from oracle.make_golden_load_fn import CASES, MODES, write_case

GOLD = json.load(open(os.path.join(GOLDEN, "load_fn.json")))
CASE_MODES = [(c, m) for c in sorted(CASES) for m in MODES]

# (h, w): landscape, portrait, square, upscaled, width already 518, exact sizes, extreme aspect ratios, odd sizes
SWEEP = [(480, 640), (500, 300), (400, 400), (60, 100), (700, 518), (392, 518), (518, 392), (518, 518), (37, 500), (500, 37),
         (1000, 999), (999, 1000), (29, 31), (203, 1001), (1001, 203), (14, 14)]


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _pillow_matches():
    import PIL
    return PIL.__version__ == GOLD["_versions"]["pillow"]


def oracle_placement(sizes, mode):
    """Output shape of the oracle and, per image, the rows and columns (top, bottom, left, right) its pixels cover.  Constant
    mid-grey images stay far below 255 after the bicubic resize, so the pixels equal to 1.0 are exactly the padding."""
    x = LO.preprocess_images([np.full((h, w, 3), 128, np.uint8) for h, w in sizes], mode)
    boxes = []
    for img in x:
        keep = (img != 1.0).any(0)
        rows, cols = np.flatnonzero(keep.any(1)), np.flatnonzero(keep.any(0))
        t, b, l, r = int(rows[0]), int(rows[-1]) + 1, int(cols[0]), int(cols[-1]) + 1
        assert keep.sum() == (b - t) * (r - l), "the image is one rectangle"
        boxes.append((t, b, l, r))
    return x.shape, boxes


class _ArgRecorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 0
        return fn


@pytest.fixture()
def dry(monkeypatch):
    """The C library replaced by a recorder, on CPU tensors (as in test_components_cpu.py)."""
    from omnivggt_official_b200 import _lib
    rec = _ArgRecorder()
    monkeypatch.setattr(_lib, "lib", lambda: rec)
    monkeypatch.setattr(_lib, "stream", lambda: 0)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(synchronize=lambda: None))
    return rec


@pytest.mark.parametrize("case,mode", CASE_MODES)
def test_oracle_matches_reference_golden(case, mode, tmp_path):
    if not _pillow_matches():
        pytest.skip("fixture hashes are for the pinned Pillow build")
    g = GOLD[case][mode]
    x = LO.load_and_preprocess_images(write_case(str(tmp_path), case), mode)
    assert list(x.shape) == g["shape"] and x.dtype == np.float32
    assert _sha(x) == g["f32_sha256"]
    assert _sha(np.rint(x.astype(np.float64) * 255).astype(np.uint8)) == g["u8_sha256"]


@pytest.mark.parametrize("mode", MODES)
def test_layout_matches_oracle_placement(mode):
    from omnivggt_official_b200 import preprocess as PP
    for sizes in [[s] for s in SWEEP] + [SWEEP, SWEEP[::-1], [(60, 100), (500, 300)]]:
        views, frame, shapes = PP.load_fn_layout(sizes, mode)
        shape, boxes = oracle_placement(sizes, mode)
        assert tuple(shape) == (len(sizes), 3) + frame
        assert (len(shapes) > 1) == (mode == "crop" and len({v[3] for v in views}) > 1)
        for (h, w), (nw, nh, crop, fh, oy, ox), box in zip(sizes, views, boxes):
            assert (nw, nh) == LO.resized_size(w, h, mode)
            assert crop == ((nh - 518) // 2 if mode == "crop" and nh > 518 else 0) and fh == min(nh, 518)
            assert (oy, oy + fh, ox, ox + nw) == box, (sizes, mode, (h, w))


@pytest.mark.parametrize("mode", MODES)
def test_errors_are_raised_before_any_device_work(dry, mode):
    from omnivggt_official_b200 import preprocess as PP
    with pytest.raises(ValueError, match="At least 1 image"):
        PP.preprocess_images([], mode)
    with pytest.raises(ValueError, match="At least 1 image"):
        PP.load_and_preprocess_images([], mode)
    with pytest.raises(ValueError, match="Mode must be"):
        PP.preprocess_images([np.zeros((30, 40, 3), np.uint8)], "resize")
    with pytest.raises(ValueError, match="Mode must be"):
        PP.load_and_preprocess_images(["never-opened.png"], "resize")
    # crop: 2000 x 10 resizes to 518 x 0; pad: the short side rounds to 0 in either orientation
    tiny = [(10, 2000)] if mode == "crop" else [(10, 2000), (2000, 10)]
    for h, w in tiny:
        im = np.zeros((h, w, 3), np.uint8)
        with pytest.raises(ValueError, match="must be > 0"):
            PP.preprocess_images([np.zeros((40, 40, 3), np.uint8), im], mode)
        with pytest.raises(ValueError):
            LO.preprocess_images([im], mode)
    assert dry.calls == []


@pytest.mark.parametrize("case,mode", CASE_MODES)
def test_dry_run_arguments(dry, case, mode, tmp_path, capsys):
    from omnivggt_official_b200 import preprocess as PP
    g = GOLD[case][mode]
    paths = write_case(str(tmp_path), case)
    out = PP.load_and_preprocess_images(paths, mode, device="cpu")
    printed = capsys.readouterr().out.strip() or None
    assert printed == g["warning"]
    assert list(out.shape) == g["shape"] and out.dtype == torch.float32
    sizes = [PP.decode_rgb(p).shape[:2] for p in sorted(paths)]
    shape, boxes = oracle_placement(sizes, mode)
    assert [n for n, _ in dry.calls] == ["ovg_preprocess_image_canvas"] * len(paths)
    for i, ((h, w), box, (_, a)) in enumerate(zip(sizes, boxes, dry.calls)):
        nw, nh = LO.resized_size(w, h, mode)
        crop = (nh - 518) // 2 if mode == "crop" and nh > 518 else 0
        assert a[1:7] == (h, w, nw, nh, crop, min(nh, 518))
        assert (a[7] is None) == (a[9] is None) == (a[15] is None) == (w == nw) and (a[10] == 0) == (w == nw)
        assert (a[11] is None) == (a[13] is None) == (h == nh) and (a[14] == 0) == (h == nh)
        assert a[16] == out[i].data_ptr() and a[17:19] == tuple(shape[2:])
        assert (a[19], a[19] + a[6], a[20], a[20] + a[3]) == box
        assert a[21] == 1.0 and a[22] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("case,mode", CASE_MODES)
def test_gpu_matches_oracle_and_golden(case, mode, tmp_path, capsys):
    from omnivggt_official_b200 import preprocess as PP
    paths = write_case(str(tmp_path), case)
    out = PP.load_and_preprocess_images(paths, mode)
    assert (capsys.readouterr().out.strip() or None) == GOLD[case][mode]["warning"]
    assert out.is_cuda and out.dtype == torch.float32
    ref = LO.load_and_preprocess_images(paths, mode)
    assert torch.equal(out.cpu(), torch.from_numpy(ref))
    if _pillow_matches():
        assert _sha(out.cpu().numpy()) == GOLD[case][mode]["f32_sha256"]


@pytest.mark.gpu
def test_canvas_places_the_image_at_an_offset():
    """ovg_preprocess_image_canvas called directly: both passes and a crop, in a wider and taller frame, fill 0.25."""
    from omnivggt_official_b200 import _lib as L
    from omnivggt_official_b200 import preprocess as PP
    lib = L.lib()
    h, w, nw, nh, crop, fh = 75, 90, 56, 84, 14, 56
    out_h, out_w, oy, ox, fill = 64, 100, 5, 37, 0.25
    im = np.random.default_rng(3).integers(0, 256, (h, w, 3), dtype=np.uint8)
    src = torch.from_numpy(im).cuda()
    hk, vk = PP.bicubic_taps(w, nw, "cuda"), PP.bicubic_taps(h, nh, "cuda")
    tmp = torch.empty(h, nw, 3, device="cuda", dtype=torch.uint8)
    out = torch.full((3, out_h, out_w), float("nan"), device="cuda")
    args = (src.data_ptr(), h, w, nw, nh, crop, fh, *(t.data_ptr() for t in hk[:3]), hk[3], *(t.data_ptr() for t in vk[:3]), vk[3],
            tmp.data_ptr(), out.data_ptr())
    L.check(lib.ovg_preprocess_image_canvas(*args, out_h, out_w, oy, ox, fill, L.stream()))
    torch.cuda.synchronize()
    want = np.full((3, out_h, out_w), fill, np.float32)
    r = PO.pil_resize_u8(im, nw, nh)[crop:crop + fh]
    want[:, oy:oy + fh, ox:ox + nw] = r.transpose(2, 0, 1).astype(np.float32) / np.float32(255)
    assert torch.equal(out.cpu(), torch.from_numpy(want))
    with pytest.raises(L.OvgError, match="does not fit"):
        L.check(lib.ovg_preprocess_image_canvas(*args, out_h, out_w, oy, out_w - nw + 1, fill, L.stream()))


@pytest.mark.gpu
def test_pad_mode_mixed_orientations_feed_the_model(tmp_path):
    from omnivggt_official_b200 import preprocess as PP
    from test_model_gpu import model
    paths = write_case(str(tmp_path), "mixed")
    images = PP.load_and_preprocess_images(paths, mode="pad")
    n = len(paths)
    assert images.shape == (n, 3, 518, 518)
    out = model("mini_conv")(images)
    torch.cuda.synchronize()
    assert out["depth"].shape == (1, n, 518, 518, 1) and out["world_points"].shape == (1, n, 518, 518, 3)
    for k in ("depth", "depth_conf", "world_points", "world_points_conf", "pose_enc"):
        assert torch.isfinite(out[k]).all(), k
