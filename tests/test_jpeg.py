"""Baseline JPEG decoding on the device (csrc/jpeg.cuh, preprocess.decode_images), bit-identical to Pillow.
CPU: the numpy oracle against Pillow over a fixture matrix (this pins the arithmetic the device reproduces to the Pillow that is
installed), the library's plan against the oracle's parse (routing, sizes, segments, unstuffed bytes), and a dry run of
decode_images with a recording stand-in for the library.  GPU: the device against Pillow over the matrix at the default and the
minimum subsequence size, camera-sized images, a batch past 2^31 bits of entropy data, a corrupted file, and both loaders on a
mixed folder.  Every fixture is encoded by Pillow at test time from a seed."""
import ctypes
import io
import os

import numpy as np
import pytest
import torch

from oracle import jpeg_oracle as J

SIZES = [(1, 1), (2, 2), (3, 5), (7, 9), (17, 33), (31, 47), (100, 75)]           # (width, height)
ENCODINGS = {
    "s444": dict(subsampling=0), "s422": dict(subsampling=1), "s420": dict(subsampling=2), "gray": dict(gray=True),
    "q1": dict(quality=1), "q50": dict(quality=50), "q90": dict(quality=90), "q100": dict(quality=100, subsampling=0),
    "optimize": dict(optimize=True), "rst1": dict(restart_marker_blocks=1), "rst3": dict(restart_marker_blocks=3, subsampling=1),
    "rstrow": dict(restart_marker_rows=1, subsampling=2),
}
BIG_ENCODINGS = ("s444", "s422", "s420", "gray", "rst3")                            # at 640 x 480


def matrix():
    """[(name, bytes)]: every size x encoding on seeded noise, and 640 x 480 octave noise for a subset of the encodings."""
    out = []
    for k, (w, h) in enumerate(SIZES):
        rgb = np.random.default_rng(k).integers(0, 256, (h, w, 3), dtype=np.uint8)
        for name, kw in ENCODINGS.items():
            out.append((f"{w}x{h}-{name}", J.encode(rgb, **kw)))
    rgb = J.octave_noise(640, 480, seed=7)
    for name in BIG_ENCODINGS:
        out.append((f"640x480-{name}", J.encode(rgb, **ENCODINGS[name])))
    return out


def routing_cases():
    """[(name, bytes, expected route)] for files that must go to the host."""
    from PIL import Image
    rgb = np.random.default_rng(11).integers(0, 256, (24, 40, 3), dtype=np.uint8)
    base = J.encode(rgb)
    cmyk = io.BytesIO()
    Image.fromarray(rgb).convert("CMYK").save(cmyk, "JPEG")
    png = io.BytesIO()
    Image.fromarray(rgb).save(png, "PNG")
    return [("progressive", J.encode(rgb, progressive=True), J.PROCESS), ("cmyk", cmyk.getvalue(), J.COLOR),
            ("truncated", base[:len(base) // 2], J.TRUNCATED), ("png", png.getvalue(), J.NOT_JPEG),
            ("short-jfif-adobe-rgb", short_jfif_adobe_rgb(), J.COLOR)]


def pillow_rgb(data: bytes) -> np.ndarray:
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def corrupted():
    """A baseline file with one byte of entropy data changed such that the data becomes inconsistent (the oracle's serial
    decode rejects it), and the same file intact."""
    rgb = J.octave_noise(96, 64, seed=5)
    data = J.encode(rgb, quality=90)
    sos = data.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big")
    for pos in range(start + 40, len(data) - 2, 7):
        if data[pos] in (0xFF, 0x00, 0xFE) or data[pos - 1] == 0xFF:
            continue
        bad = bytearray(data)
        bad[pos] ^= 0xFF
        bad = bytes(bad)
        p = J.parse(bad)
        if p.route != J.DEVICE:
            continue
        try:
            J.huffman_decode(p)
        except ValueError:
            return bad, data
    raise AssertionError("no inconsistent single-byte corruption found")


def dqt_patched():
    """A quality-100 4:4:4 file whose quantisation tables are overwritten with 40: the entropy data stays consistent, but the
    dequantised blocks leave the range where libjpeg-turbo's C and SIMD IDCTs agree (Pillow runs the SIMD one)."""
    data = bytearray(J.encode(J.octave_noise(64, 48, seed=9), quality=100, subsampling=0))
    i = 2
    while data[i + 1] != 0xDA:
        ln = int.from_bytes(data[i + 2:i + 4], "big")
        if data[i + 1] == 0xDB:
            k = i + 4
            while k < i + 2 + ln:
                assert data[k] >> 4 == 0, "8-bit tables"
                data[k + 1:k + 65] = bytes([40]) * 64
                k += 65
        i += 2 + ln
    return bytes(data)


def short_jfif_adobe_rgb():
    """A JFIF APP0 shorter than libjpeg's 14 bytes (so not seen as JFIF) and an Adobe APP14 with transform 0: libjpeg treats the
    three components as RGB, so the file goes to the host."""
    data = J.encode(np.random.default_rng(12).integers(0, 256, (16, 16, 3), dtype=np.uint8))
    assert data[2:4] == b"\xff\xe0"
    rest = data[4 + int.from_bytes(data[4:6], "big"):]
    adobe = b"Adobe" + bytes([0, 100, 0, 0, 0, 0, 0])
    return data[:2] + b"\xff\xe0\x00\x07JFIF\x00" + b"\xff\xee" + (2 + len(adobe)).to_bytes(2, "big") + adobe + rest


def _write(d, files):
    paths = []
    for name, data in files:
        p = os.path.join(d, name + (".png" if data[:4] == b"\x89PNG" else ".jpg"))
        with open(p, "wb") as f:
            f.write(data)
        paths.append(p)
    return paths


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name,data", matrix(), ids=lambda v: v if isinstance(v, str) else "")
def test_oracle_matches_pillow(name, data):
    p = J.parse(data)
    assert p.route == J.DEVICE, J.REASONS[p.route]
    got, want = J.decode(data), pillow_rgb(data)
    assert got.shape == want.shape and np.array_equal(got, want), name


def test_routing_cases_go_to_the_host():
    for name, data, route in routing_cases():
        assert J.parse(data).route == route, name


def test_oracle_flags_a_block_outside_the_idct_range():
    data = dqt_patched()
    p = J.parse(data)
    assert p.route == J.DEVICE
    J.huffman_decode(p)                                  # consistent entropy data
    with pytest.raises(ValueError, match="C and SIMD"):
        J.decode(data)


def test_plan_matches_oracle_parse():
    from omnivggt_official_b200 import _lib as L
    files = matrix() + [(n, d) for n, d, _ in routing_cases()]
    bad, _ = corrupted()
    files += [("corrupted", bad), ("dqt-patched", dqt_patched())]
    plan = L.JpegPlan([d for _, d in files])
    stream = np.zeros(plan.stream_bytes, np.uint8)
    plan.fill_stream(stream.ctypes.data)
    segs = plan.segments()
    it = iter(segs)
    for i, (name, data) in enumerate(files):
        p = J.parse(data)
        route, h, w, nc = plan.files[i]
        assert route == p.route, (name, route, p.route)
        if route != J.DEVICE:
            continue
        assert (h, w, nc) == (p.height, p.width, len(p.comps)), name
        _, _, mx, my = p.mcu_geometry
        per = p.restart or mx * my
        for k, seg in enumerate(p.segments):
            f, off, nb, m0, nm = next(it)
            assert (f, nb, m0, nm) == (i, len(seg), k * per, min(per, mx * my - k * per)), (name, k)
            assert off % 16 == 0 and stream[off:off + nb].tobytes() == seg, (name, k)
            assert not stream[off + nb:off + nb + 16].any(), "zero padding after every segment"
    assert next(it, None) is None
    assert plan.subsequences >= len(segs)


def test_plan_rejects_a_subsequence_size_below_the_minimum():
    from omnivggt_official_b200 import _lib as L
    data = J.encode(J.octave_noise(64, 64, seed=2))
    bits = 8 * L.JpegPlan([data]).segments()[0][2]
    assert L.JpegPlan([data], L.JPEG_MIN_SUBSEQ_BITS).subsequences == -(-bits // L.JPEG_MIN_SUBSEQ_BITS)
    with pytest.raises(L.OvgError, match="subseq_bits"):
        L.JpegPlan([data], L.JPEG_MIN_SUBSEQ_BITS - 1)


class _DecodeRecorder:
    """Stands in for the library's compute entry points: records the calls and sets the status word of the files in `flag`."""

    def __init__(self, flag=()):
        self.calls, self.flag = [], set(flag)

    def ovg_jpeg_decode(self, plan, stream, ptrs, status, ws, wsb, st):
        self.calls.append(("ovg_jpeg_decode", [ptrs[i] for i in range(len(ptrs))], wsb))
        n = len(ptrs)
        st_arr = (ctypes.c_int32 * n).from_address(status)
        for i in self.flag:
            st_arr[i] = 1
        self.ptrs = [ptrs[i] for i in range(n)]
        return 0


def test_dry_run_routing_fallback_and_order(monkeypatch, tmp_path):
    from omnivggt_official_b200 import _lib as L
    from omnivggt_official_b200 import preprocess as PP
    rgb = J.octave_noise(40, 24, seed=3)
    files = [("a-base", J.encode(rgb)), ("b-prog", J.encode(rgb, progressive=True)), ("c-gray", J.encode(rgb, gray=True)),
             ("d-png", dict((n, d) for n, d, _ in routing_cases())["png"]), ("e-flagged", J.encode(rgb[:16], quality=60))]
    paths = _write(str(tmp_path), files)
    rec = _DecodeRecorder(flag={4})
    monkeypatch.setattr(L, "lib", lambda: rec)
    monkeypatch.setattr(L, "stream", lambda: 0)
    out = PP.decode_images(paths, device="cpu")
    assert [c[0] for c in rec.calls] == ["ovg_jpeg_decode"]
    on_device = [i for i, p in enumerate(rec.ptrs) if p]
    assert on_device == [0, 2, 4]
    for i, (p, t) in enumerate(zip(paths, out)):
        want = PP.decode_rgb(p)
        assert t.dtype == torch.uint8 and tuple(t.shape) == want.shape
        if i in (0, 2):                                  # device outputs: the stand-in wrote nothing into them
            assert t.data_ptr() == rec.ptrs[i]
        else:                                            # host-routed, or flagged: Pillow's pixels
            assert np.array_equal(t.numpy(), want), i


# ------------------------------------------------------------------------------------------------------------------ GPU
def _device_decode(tmp_path, files, subseq_bits=0):
    from omnivggt_official_b200 import preprocess as PP
    return PP.decode_images(_write(str(tmp_path), files), subseq_bits=subseq_bits)


@pytest.mark.gpu
@pytest.mark.parametrize("subseq", ["default", "minimum"])
def test_gpu_matrix_equals_pillow(subseq, tmp_path):
    from omnivggt_official_b200 import _lib as L
    files = matrix()
    out = _device_decode(tmp_path, files, 0 if subseq == "default" else L.JPEG_MIN_SUBSEQ_BITS)
    for (name, data), t in zip(files, out):
        assert t.is_cuda and np.array_equal(t.cpu().numpy(), pillow_rgb(data)), name


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,quality,subsampling", [(6048, 4032, 95, 1), (4032, 3024, 90, 2)])
def test_gpu_camera_sized_equals_pillow(w, h, quality, subsampling, tmp_path):
    from omnivggt_official_b200 import _lib as L
    data = J.encode(J.octave_noise(w, h, seed=w), quality=quality, subsampling=subsampling)
    plan = L.JpegPlan([data])
    assert plan.files[0][0] == J.DEVICE
    t = _device_decode(tmp_path, [("cam", data)])[0]
    assert np.array_equal(t.cpu().numpy(), pillow_rgb(data))


@pytest.mark.gpu
def test_gpu_batch_past_2_31_bits(tmp_path):
    """24 views of 6048 x 4032 at quality 95, 4:2:2: the entropy data of the batch passes 2^31 bits (64-bit offsets)."""
    from omnivggt_official_b200 import _lib as L
    data = J.encode(J.octave_noise(6048, 4032, seed=1), quality=95, subsampling=1)
    files = [(f"v{i:02d}", data) for i in range(24)]
    plan = L.JpegPlan([d for _, d in files])
    bits = 8 * sum(nb for _, _, nb, _, _ in plan.segments())
    assert bits > 2 ** 31, bits
    out = _device_decode(tmp_path, files)
    want = torch.from_numpy(pillow_rgb(data)).cuda()
    for i, t in enumerate(out):
        assert torch.equal(t, want), i


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["entropy", "idct-range"])
def test_gpu_flagged_file_equals_pillow(kind, tmp_path):
    """A file with inconsistent entropy data, and one with a block outside the IDCT range where libjpeg-turbo's C and SIMD paths
    agree: the status word is set and decode_images returns Pillow's pixels; an intact file in the same batch is not flagged."""
    from omnivggt_official_b200 import _lib as L
    bad, good = corrupted() if kind == "entropy" else (dqt_patched(), corrupted()[1])
    plan = L.JpegPlan([bad, good])
    stream = torch.empty(plan.stream_bytes, dtype=torch.uint8, pin_memory=True)
    plan.fill_stream(stream.data_ptr())
    d_stream = stream.cuda()
    ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device="cuda")
    outs = [torch.empty(plan.files[i][1], plan.files[i][2], 3, dtype=torch.uint8, device="cuda") for i in range(2)]
    ptrs = (ctypes.c_void_p * 2)(*[o.data_ptr() for o in outs])
    status = torch.full((2,), -1, dtype=torch.int32, device="cuda")
    L.check(L.lib().ovg_jpeg_decode(plan.handle, d_stream.data_ptr(), ptrs, status.data_ptr(), ws.data_ptr(),
                                    plan.workspace_bytes, L.stream()))
    st = status.cpu().tolist()
    assert st[0] != 0 and st[1] == 0, st
    assert (st[0] == 16) == (kind == "idct-range"), st
    assert np.array_equal(outs[1].cpu().numpy(), pillow_rgb(good))
    got = _device_decode(tmp_path, [("bad", bad), ("good", good)])
    assert np.array_equal(got[0].cpu().numpy(), pillow_rgb(bad))
    assert np.array_equal(got[1].cpu().numpy(), pillow_rgb(good))


def _mixed_folder(d, heights_to_518=False):
    """PNG, RGBA PNG, progressive, gray and baseline JPEGs of different sizes.  heights_to_518: every size resizes to the same
    height at width 518 (load_images_and_cameras stacks the views)."""
    from PIL import Image
    sizes = [(1036, 700), (777, 525), (518, 350), (259, 175), (1554, 1050), (1036, 700)] if heights_to_518 else \
            [(640, 480), (480, 640), (300, 300), (1001, 203), (97, 131), (800, 600)]
    os.makedirs(d, exist_ok=True)
    for i, (w, h) in enumerate(sizes):
        rgb = J.octave_noise(w, h, seed=20 + i)
        p = os.path.join(d, f"view-{i}")
        if i == 0:
            Image.fromarray(rgb).save(p + ".png")
        elif i == 1:
            a = np.concatenate([rgb, (np.arange(w)[None, :, None] % 256).repeat(h, 0).astype(np.uint8)], -1)
            Image.fromarray(a, "RGBA").save(p + ".png")
        else:
            kw = [dict(progressive=True), dict(gray=True), dict(quality=90, subsampling=2),
                  dict(quality=95, subsampling=1, restart_marker_rows=2)][i - 2]
            with open(p + ".jpg", "wb") as f:
                f.write(J.encode(rgb, **kw))
    return sorted(os.path.join(d, f) for f in os.listdir(d))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["crop", "pad"])
def test_gpu_load_and_preprocess_images_mixed_folder(mode, tmp_path):
    from omnivggt_official_b200 import preprocess as PP
    paths = _mixed_folder(str(tmp_path / "imgs"))
    got = PP.load_and_preprocess_images(paths, mode)
    want = PP.preprocess_images([PP.decode_rgb(p) for p in sorted(paths)], mode)
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_gpu_load_images_and_cameras_mixed_folder(tmp_path):
    from omnivggt_official_b200 import preprocess as PP
    paths = _mixed_folder(str(tmp_path / "imgs"), heights_to_518=True)
    got = PP.load_images_and_cameras(str(tmp_path / "imgs"))
    want = PP.preprocess_views([PP.decode_rgb(p) for p in paths])
    for a, b in zip(got[:5], want[:5]):
        assert torch.equal(a, b)
    assert got[5:] == want[5:]
