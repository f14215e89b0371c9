"""Model-free sky segmentation (reference omnivggt/viz.py:357-393 segment_sky) and the --mask_sky confidence of the GLB export
(visual_util.py:140-188).
CPU: the numpy oracle against the UNMODIFIED reference's outputs (tests/golden/sky.safetensors), its HSV and colour test against
cv2 over every colour, its opening against scipy and its component selection against cv2, a dry run of the library calls, and
the errors.
GPU: libovg's ovg_segment_sky through geometry.segment_sky and OmniVGGT.sky_mask against the oracle bit for bit, large and
adversarial masks, repeats, and mask_sky on point_cloud / mesh / matches and the mini model."""
import os

import numpy as np
import pytest
import torch
from safetensors.torch import load_file

from conftest import GOLDEN
from oracle import sky_oracle as SO
from oracle.make_golden_cloud import GLB_CASES
from oracle.make_golden_sky import ground, make_cases, sky_cloud_inputs
from ovg_support import dry, scene, sha256  # noqa: F401  (fixture)

GOLD = {k: v.numpy() for k, v in load_file(os.path.join(GOLDEN, "sky.safetensors")).items()}
CASES = make_cases()
NAMES = sorted(CASES)


def _bits_sha(mask) -> bytes:
    return sha256(np.packbits(np.ascontiguousarray(mask, dtype=bool)), hex=False)


def _check_golden(name, mask):
    assert int(mask.sum()) == int(GOLD[f"{name}_count"]) and _bits_sha(mask) == GOLD[f"{name}_sha256"].tobytes(), name


def _check_glb_golden(i, points, colors):
    """A cloud against the reference's GLB export of case i; an empty cloud is its placeholder (visual_util.py:226-229)."""
    if len(points) == 0:
        points, colors = np.array([[1, 0, 0]]), np.array([[255, 255, 255]])
    assert len(points) == int(GOLD[f"glb{i}_count"]), i
    assert sha256(points, hex=False) == GOLD[f"glb{i}_points_sha256"].tobytes(), i
    assert sha256(colors, hex=False) == GOLD[f"glb{i}_colors_sha256"].tobytes(), i


def _source(g, src):
    return (g["world_points_from_depth"], g["depth_conf"]) if src == "depth" else (g["world_points"], g["world_points_conf"])


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference_golden(name):
    _check_golden(name, SO.segment_sky(CASES[name]))


def test_cases_cover_the_contract():
    assert {CASES[n].dtype for n in NAMES} == {np.dtype(np.uint8), np.dtype(np.float32), np.dtype(np.float64)}
    assert any(CASES[n].min() < 0 for n in NAMES) and any(CASES[n].max() > 1 for n in NAMES if CASES[n].dtype != np.uint8)
    assert int(GOLD["no_sky_count"]) == 0 and int(GOLD["all_sky_count"]) == 33 * 45
    assert int(GOLD["tiny_4x4_count"]) == 0 and int(GOLD["tiny_5x5_count"]) == 25
    assert int(GOLD["checkerboard_count"]) == 0
    from scipy import ndimage
    cb = SO.color_mask(CASES["checkerboard"])                   # one 8-connected component before the opening
    assert ndimage.label(cb, structure=np.ones((3, 3)))[1] == 1 and not SO.opening(cb).any()


def test_oracle_views_and_glb_clouds_match_reference_golden():
    g = sky_cloud_inputs()
    assert sha256(g["images"], hex=False) == GOLD["images_sha256"].tobytes()
    sky = SO.sky_of_views(g["images"])
    assert _bits_sha(sky) == GOLD["views_sky_sha256"].tobytes() and sky.any()
    for i, (src, pct, frame, black, white) in enumerate(GLB_CASES):
        world, conf = _source(g, src)
        o = SO.point_cloud(world, conf, g["images"], g["extrinsic"], sky, pct, 1e-5, frame, black, white)
        _check_glb_golden(i, o["points"], o["colors"])
        assert float(o["conf_threshold"]) == float(GOLD[f"glb{i}_thr"]), i


def test_oracle_hsv_and_colour_test_match_cv2_on_every_colour():
    cv2 = pytest.importorskip("cv2")
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    hsv = cv2.cvtColor(img, cv2.COLOR_BGR2HSV)
    assert np.array_equal(SO.bgr2hsv(img), hsv)
    m = cv2.inRange(hsv, np.array([0, 0, 100]), np.array([30, 255, 255])).view(bool)
    m |= (hsv[:, :, 1] < 10) & (hsv[:, :, 2] > 150)
    m |= (hsv[:, :, 1] < 30) & (hsv[:, :, 2] > 180)
    m |= (hsv[:, :, 1] < 50) & (hsv[:, :, 2] > 220)
    assert np.array_equal(SO.color_mask(img), m)


def _random_masks():
    rng = np.random.default_rng(5)
    from scipy import ndimage
    out = [rng.random((h, w)) < p for h, w, p in ((1, 1, 1.0), (1, 7, 0.9), (6, 1, 0.9), (4, 4, 1.0), (5, 5, 1.0), (5, 6, 0.95),
                                                  (7, 5, 0.9), (9, 9, 0.8))]
    for k in range(12):
        h, w = rng.integers(5, 90, 2)
        out.append(ndimage.uniform_filter(rng.random((h, w)), int(rng.integers(1, 8))) > rng.uniform(0.3, 0.7))
        out.append(rng.random((h, w)) < rng.uniform(0.5, 0.97))
    return out


def test_oracle_opening_matches_scipy():
    from scipy import ndimage
    for m in _random_masks():
        assert np.array_equal(SO.opening(m), ndimage.binary_opening(m, structure=np.ones((5, 5)))), m.shape


def test_oracle_selection_matches_cv2_components():
    cv2 = pytest.importorskip("cv2")
    for m in _random_masks():
        for mask in (m, SO.opening(m)):
            _, labels, stats, _ = cv2.connectedComponentsWithStats(mask.astype(np.uint8), connectivity=8)
            sizes = stats[1:, cv2.CC_STAT_AREA]
            order = sizes.argsort()[::-1]
            sel = [1 + o for o in order if sizes[o] > sizes[order[0]] / 2]
            assert np.array_equal(SO.select_components(mask), np.isin(labels, sel)), mask.shape


def test_dry_run_launches_do_not_depend_on_views(dry, monkeypatch):
    from omnivggt_official_b200 import OmniVGGT, geometry
    monkeypatch.setattr(geometry, "_device_of", lambda *xs: torch.device("cpu"))
    seqs = []
    for S in (1, 24):
        dry.calls.clear()
        sky = OmniVGGT.sky_mask(scene(S, 6, 8))
        assert sky.shape == (S, 6, 8) and sky.dtype == torch.bool
        assert dry.names() == ["ovg_sky_workspace_bytes", "ovg_segment_sky"]
        a = dry.calls[1][1]
        assert a[1:8] == (0, 3 * 6 * 8, 1, 6 * 8, S, 6, 8) and a[8] is None     # fp32 [S,3,H,W] read in place
        seqs.append(dry.names())
    assert seqs[0] == seqs[1] and len(dry.reads) == 0
    dry.calls.clear()
    geometry.segment_sky(np.zeros((5, 7, 3), np.uint8))
    assert dry.calls[1][1][1:8] == (1, 5 * 7 * 3, 3, 1, 1, 5, 7)
    dry.calls.clear()
    geometry.segment_sky(torch.zeros(5, 7, 3, dtype=torch.float64))           # fp64 -> uint8 by torch, then the uint8 path
    assert dry.calls[1][1][1] == 1


def _host_syncs(monkeypatch):
    n = [0]
    item, cpu = torch.Tensor.item, torch.Tensor.cpu

    def count(fn):
        def wrapped(self, *a, **k):
            n[0] += 1
            return fn(self, *a, **k)
        return wrapped

    monkeypatch.setattr(torch.Tensor, "item", count(item))
    monkeypatch.setattr(torch.Tensor, "cpu", count(cpu))
    return n


@pytest.mark.parametrize("method", ["point_cloud", "mesh", "matches"])
def test_dry_run_mask_sky_adds_no_host_read_and_false_adds_no_launch(dry, monkeypatch, method):
    from omnivggt_official_b200 import OmniVGGT, ops
    monkeypatch.setattr(ops, "point_cloud_count", lambda *a, **k: torch.zeros((), dtype=torch.int64))
    monkeypatch.setattr(ops.Matcher, "counts", lambda self: ([0] * self.P, False))
    syncs = _host_syncs(monkeypatch)
    fn = getattr(OmniVGGT, method)
    pred = scene(3, 6, 8)
    base = None
    for mask_sky in (False, True, torch.zeros(3, 6, 8, dtype=torch.bool), torch.zeros(1, 3, 6, 8, dtype=torch.bool)):
        dry.calls.clear()
        syncs[0] = 0
        fn(pred, mask_sky=mask_sky)
        names = dry.names()
        if base is None:
            base = (names, syncs[0])
            assert not any("sky" in n for n in names)
            continue
        assert syncs[0] == base[1]
        sky_calls = ["ovg_sky_workspace_bytes", "ovg_segment_sky"] if mask_sky is True else ["ovg_sky_mask_conf"]
        assert names == sky_calls + base[0]                             # the sky comes before the percentile
        if mask_sky is True:
            assert dry.calls[1][1][5] == 3 and dry.calls[1][1][8] is not None   # every view, with the confidence
    dry.calls.clear()
    OmniVGGT.point_cloud(pred, mask_sky=True, frame=2)
    assert dry.calls[1][1][5] == 3                                      # the sky multiplies all views, then the frame is taken


def test_errors_before_any_device_work(dry, monkeypatch):
    from omnivggt_official_b200 import OmniVGGT, geometry
    monkeypatch.setattr(geometry, "_device_of", lambda *xs: torch.device("cpu"))
    pred = scene(3, 6, 8)
    for bad in (np.zeros((4, 5)), np.zeros((4, 5, 4)), np.zeros((2, 4, 5, 3)), torch.zeros(3, 4, 5)):
        with pytest.raises(ValueError, match="shape"):
            geometry.segment_sky(bad)
    for dt in (np.int32, np.float16, np.int64, bool):
        with pytest.raises(ValueError, match="dtype"):
            geometry.segment_sky(np.zeros((4, 5, 3), dt))
    with pytest.raises(ValueError, match="dtype"):
        geometry.segment_sky(torch.zeros(4, 5, 3, dtype=torch.bfloat16))
    for fn in (OmniVGGT.point_cloud, OmniVGGT.mesh, OmniVGGT.matches):
        for bad in (torch.zeros(3, 6, 8, dtype=torch.uint8), torch.zeros(3, 6, 8), np.zeros((3, 6, 8), bool), "yes", 1, None):
            with pytest.raises(ValueError, match="mask_sky"):
                fn(pred, mask_sky=bad)
        for shape in ((2, 6, 8), (3, 8, 6), (3, 6, 8, 1), (2, 3, 6, 8), (6, 8)):
            with pytest.raises(ValueError, match="mask_sky"):
                fn(pred, mask_sky=torch.zeros(shape, dtype=torch.bool))
        with pytest.raises(ValueError, match="mask_sky"):
            fn(pred, mask_sky=torch.zeros(3, 6, 8, dtype=torch.bool, device="meta"))
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
def _hwc_f32(img):
    """A case as fp32 [H, W, 3] for the model path (uint8 / 255 and float64 rounded to fp32: the oracle sees the same)."""
    if img.dtype == np.uint8:
        return img.astype(np.float32) / np.float32(255)
    return img.astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_drop_in_and_sky_mask_match_oracle_and_golden(name):
    from omnivggt_official_b200 import OmniVGGT, geometry
    img = CASES[name]
    d = geometry.segment_sky(img)
    assert d.is_cuda and d.dtype == torch.bool and d.shape == img.shape[:2]
    _check_golden(name, d.cpu().numpy())
    for arg in (torch.from_numpy(img), torch.from_numpy(img).cuda()):
        assert torch.equal(geometry.segment_sky(arg), d)
    f = _hwc_f32(img)
    views = np.stack([f, f[::-1, ::-1], np.roll(f, 3, axis=1)])                # three views in one call: no label crosses views
    images = torch.from_numpy(np.ascontiguousarray(views.transpose(0, 3, 1, 2))).cuda()
    got = OmniVGGT.sky_mask({"images": images[None]}).cpu().numpy()
    assert np.array_equal(got, np.stack([SO.segment_sky(np.ascontiguousarray(v)) for v in views]))


def _blob_images(S, H, W, seed, cell=24):
    """fp32 [S, 3, H, W]: sky-coloured and ground blobs from upsampled noise, with bright grey clouds."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(S, 1, H // cell + 2, W // cell + 2, generator=g)
    field = torch.nn.functional.interpolate(lo, size=(H, W), mode="bilinear", align_corners=False)[:, 0]
    y = torch.arange(H, dtype=torch.float32)[:, None] / H
    sky = torch.stack([0.27 + 0.3 * y, 0.5 + 0.2 * y, 0.92 - 0.1 * y]).expand(3, H, W)
    ground = torch.rand(S, 3, H, W, generator=g) * 0.38
    img = torch.where((field > 0.55)[:, None], sky[None], ground)
    cloud = (field > 0.8)[:, None] & (torch.rand(S, 1, H, W, generator=g) < 0.98)
    return torch.where(cloud, torch.full_like(img, 0.88), img).contiguous()


def _check_views(images):
    from omnivggt_official_b200 import OmniVGGT
    d = OmniVGGT.sky_mask({"images": images.cuda()})
    h = images.numpy()
    for f in range(len(h)):
        assert np.array_equal(d[f].cpu().numpy(), SO.segment_sky(np.ascontiguousarray(h[f].transpose(1, 2, 0)))), f
    return d


@pytest.mark.gpu
def test_24_views_518_and_two_12mp_views_match_oracle_and_repeat():
    from omnivggt_official_b200 import OmniVGGT, _lib
    lib = _lib.load()
    images = _blob_images(24, 518, 518, 1)
    n0 = lib.ovg_launch_count()
    d = _check_views(images)
    n1 = lib.ovg_launch_count()
    OmniVGGT.sky_mask({"images": images[:1].cuda()})
    n2 = lib.ovg_launch_count()
    assert n1 - n0 == n2 - n1                                           # launches do not depend on the number of views
    assert 0.1 < d.float().mean().item() < 0.6
    for _ in range(3):
        assert torch.equal(OmniVGGT.sky_mask({"images": images.cuda()}), d)
    big = _blob_images(2, 3024, 4032, 2, cell=300)
    db = _check_views(big)
    assert torch.equal(OmniVGGT.sky_mask({"images": big.cuda()}), db) and db.any()


def _labelling_worst_cases(H=518, W=518):
    """(name, sky bool [H, W]) masks whose opening is themselves: 5-px-wide structures."""
    out = []
    m = np.zeros((H, W), bool)                                          # serpentine: 5-px rows joined at alternate ends
    for k, y in enumerate(range(0, H - 5, 10)):
        m[y:y + 5, :] = True
        if y + 10 < H - 5:
            x = W - 5 if k % 2 == 0 else 0
            m[y:y + 15, x:x + 5] = True
    out.append(("serpentine", m))
    m = np.zeros((H, W), bool)                                          # square spiral, 5-px arms, 5-px gaps
    t, l, b, r = 0, 0, H, W
    while b - t >= 5 and r - l >= 5:
        m[t:t + 5, l:r] = True
        m[t:b, r - 5:r] = True
        m[b - 5:b, l:r] = True
        if b - t > 25:
            m[t + 10:b, l:l + 5] = True
        t, l, b, r = t + 10, l + 10, b - 10, r - 10
        if b - t >= 5 and r - l >= 5:
            m[t - 5:t, l - 5:l + 5] = True                               # joins the next ring: one spiral
    out.append(("spiral", m))
    out.append(("everything", np.ones((H, W), bool)))
    m = np.zeros((H, W), bool)                                          # 5x5 blocks touching only at their corners
    for k in range(0, min(H, W) - 5, 5):
        m[k:k + 5, k:k + 5] = True
        m[k:k + 5, (W - 5 - k):(W - k)] = True
    out.append(("diagonal_chains", m))
    m = np.zeros((H, W), bool)                                          # thousands of equal 5x5 components
    for y in range(0, H - 5, 7):
        for x in range(0, W - 5, 7):
            m[y:y + 5, x:x + 5] = True
    out.append(("equal_components", m))
    return out


@pytest.mark.gpu
def test_labelling_worst_cases_match_oracle():
    from omnivggt_official_b200 import geometry
    for name, m in _labelling_worst_cases():
        img = ground(*m.shape, 40)
        img[m] = (120, 160, 240)                                         # sky-coloured everywhere in the image
        o = SO.segment_sky(img)
        d = geometry.segment_sky(img).cpu().numpy()
        assert np.array_equal(d, o), name
        if name != "equal_components":
            assert np.array_equal(SO.opening(m), m) and o.any(), name
    from scipy import ndimage
    _, m = _labelling_worst_cases()[-1]
    assert ndimage.label(m)[1] > 5000 and int(o.sum()) == int(m.sum())


def _pred(g, device="cuda"):
    keys = ("images", "extrinsic", "world_points_from_depth", "depth_conf", "world_points", "world_points_conf")
    return {k: torch.from_numpy(np.ascontiguousarray(g[k]))[None].to(device) for k in keys}


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(GLB_CASES)))
def test_point_cloud_mask_sky_matches_reference_golden(i):
    from omnivggt_official_b200 import OmniVGGT
    g = sky_cloud_inputs()
    src, pct, frame, black, white = GLB_CASES[i]
    world, conf = _source(g, src)
    pred = _pred(g)
    d = OmniVGGT.point_cloud(pred, source=src, conf_percent=pct, frame=frame, mask_black_bg=black, mask_white_bg=white,
                             mask_sky=True)
    sky = SO.sky_of_views(g["images"])
    assert float(d["conf_threshold"]) == float(GOLD[f"glb{i}_thr"])
    o = SO.point_cloud(world, conf, g["images"], g["extrinsic"], sky, pct, 1e-5, frame, black, white)
    for k in ("points", "colors", "frame"):
        assert np.array_equal(d[k].cpu().numpy(), o[k]), (i, k)
    _check_glb_golden(i, d["points"].cpu().numpy(), d["colors"].cpu().numpy())
    explicit = OmniVGGT.point_cloud(pred, source=src, conf_percent=pct, frame=frame, mask_black_bg=black, mask_white_bg=white,
                                    mask_sky=OmniVGGT.sky_mask(pred))
    for k in d:
        assert torch.equal(d[k], explicit[k]), k


@pytest.mark.gpu
def test_mesh_and_matches_mask_sky_match_oracle_composition():
    from omnivggt_official_b200 import OmniVGGT
    g = sky_cloud_inputs()
    pred = _pred(g)
    sky = SO.sky_of_views(g["images"])
    sky_t = torch.from_numpy(sky).cuda()
    assert torch.equal(OmniVGGT.sky_mask(pred), sky_t)
    for layout in ("reference", "glb"):
        for frame in (None, 1):
            d = OmniVGGT.mesh(pred, conf_percent=30.0, frame=frame, mask_white_bg=True, layout=layout, mask_sky=True)
            o = SO.mesh(g["world_points_from_depth"], g["depth_conf"], g["images"], g["extrinsic"], sky, 30.0, 1e-5, frame,
                        False, True, layout)
            for k in (("vertices", "face_colors", "faces") if layout == "reference" else ("positions", "colors", "indices")):
                assert np.array_equal(d[k].cpu().numpy(), o[k]), (layout, frame, k)
            e = OmniVGGT.mesh(pred, conf_percent=30.0, frame=frame, mask_white_bg=True, layout=layout, mask_sky=sky_t[None])
            for k in d:
                assert torch.equal(d[k], e[k]), k
    masked = dict(pred)
    masked["depth_conf"] = torch.from_numpy(SO.mask_conf(g["depth_conf"], sky))[None].cuda()
    a = OmniVGGT.matches(pred, conf_percent=20.0, mask_sky=True)
    b = OmniVGGT.matches(masked, conf_percent=20.0)
    c = OmniVGGT.matches(pred, conf_percent=20.0, mask_sky=sky_t)
    assert len(a) == 3 and sum(m["count"] for m in a) > 0
    for x, y, z in zip(a, b, c):
        assert x["count"] == y["count"] == z["count"]
        assert torch.equal(x["xy_i"], y["xy_i"]) and torch.equal(x["xy_j"], y["xy_j"]) and torch.equal(x["xy_j"], z["xy_j"])
    full = OmniVGGT.point_cloud(pred, conf_percent=0.0)
    cut = OmniVGGT.point_cloud(pred, conf_percent=0.0, mask_sky=True)
    assert len(cut["points"]) < len(full["points"])


@pytest.mark.gpu
def test_mask_sky_conf_multiply_is_fp32_exact():
    from omnivggt_official_b200 import ops
    conf = torch.tensor([1.5, -2.0, float("inf"), float("nan"), 0.0, 3e-39, -0.0, 7.0], device="cuda")
    sky = torch.tensor([1, 1, 1, 1, 1, 1, 0, 0], dtype=torch.bool, device="cuda")
    got = ops.sky_mask_conf(conf, sky.view(torch.uint8)).cpu().numpy()
    with np.errstate(invalid="ignore"):                                  # inf * 0
        want = SO.mask_conf(conf.cpu().numpy(), sky.cpu().numpy())
    assert np.array_equal(got, want, equal_nan=True)
    ok = ~np.isnan(want)
    assert np.array_equal(got[ok].view(np.uint32), want[ok].view(np.uint32))        # -2 * 0 = -0, as numpy multiplies


@pytest.mark.gpu
def test_model_point_cloud_mask_sky():
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
    img = inp["images"]
    img[0, :, :, :20] = torch.tensor([0.3, 0.55, 0.92], device="cuda")[None, :, None, None]     # a sky band in every view
    pred = m.postprocess(m(depth_gt_index=[1], camera_gt_index=[0], **inp))
    sky = m.sky_mask(pred)
    assert sky.shape == (3, 56, 56) and sky[:, :20].all()
    images = pred["images"][0].float().cpu().numpy()
    assert np.array_equal(sky.cpu().numpy(), SO.sky_of_views(images))
    d = m.point_cloud(pred, conf_percent=25.0, conf_floor=0.1, mask_sky=True)
    world = pred["world_points_from_depth"][0].cpu().numpy()
    conf = pred["depth_conf"][0].cpu().numpy()
    ext = pred["extrinsic"][0].cpu().numpy()
    o = SO.point_cloud(world, conf, images, ext, sky.cpu().numpy(), 25.0, 0.1)
    for k in ("points", "colors", "frame"):
        assert np.array_equal(d[k].cpu().numpy(), o[k]), k
    assert len(d["points"]) > 0 and not (d["frame"] < 0).any()
