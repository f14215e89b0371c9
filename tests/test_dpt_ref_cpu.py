"""The DPT references of oracle/kernel_ref.py on the CPU: fp32 emulations of the fused output tail and of the upsampling kernel
pass their bounds, emulations with one seeded mistake fail them at the row or column of the mistake, and the fused tail's strip
geometry holds for every shape ovg_dpt_tail_supported accepts."""
import re

import numpy as np
import pytest
import torch

from oracle import kernel_ref as R

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64


def _fma(a, b, c):
    """fp32 fma(a, b, c): the product is exact in fp64, the sum rounded once there and once to fp32 (within the bounds)."""
    return (a.double() * b.double() + c.double()).float()


def _store16(x, dtype):
    return (x.clamp(-65504.0, 65504.0) if dtype == F16 else x).to(dtype).float()


def _failure(checks):
    """Run the checks in turn; the first AssertionError message, or None if all pass."""
    for c in checks:
        try:
            c()
        except AssertionError as e:
            return str(e)
    return None


def _at(msg, dim):
    m = re.search(rf"\b{dim}=(\d+)", msg)
    return int(m.group(1)) if m else None


# ----------------------------------------------------------------------------------------------- fused tail
def _emulate_tail(src, tx, ty, w3x3, bias, w2, b2, head_act, H, W, dtype, sms=132, mistake=None):
    """fusedtail_kernel in fp32 on the CPU, one CTA walking every work item in order: 128-pixel strips, segments with their two
    halo rows, the producers' itab walk and fmul2 / ffma2 blends rounded to 16 bits into a two-stage A buffer (zero columns left
    and right of the image), the row-by-row accumulation of the three kernel rows, and the epilogue with the table classes.
    `mistake` seeds one error: "halo" (a segment starts at its first output row, without the input row above it), "zero_col"
    (the zero column right of the image is not written), "row_class" (the border rows take the interior table class), "itab"
    (one strip pixel is assigned to the neighbouring source interval), "conf" (no 1 + in the confidence)."""
    Fr, h, w, C = src.shape
    sch = R.tail_schedule(Fr, H, W, sms)
    sy = np.float32(h - 1) / np.float32(H - 1)
    sx = np.float32(w - 1) / np.float32(W - 1)
    wk = w3x3.float().reshape(32, 3, 3, 128)
    wcat = torch.cat([torch.cat([wk[:, ky, kx] for kx in range(3)], 1) for ky in (2, 1, 0)], 0).t()    # [384, 96]
    src32 = src.float()
    gx = gy = None
    if tx is not None:
        gx, gy = (t.float() for t in R.tail_tables_ref(tx, ty, w3x3, H, W))
    preds = torch.full((Fr, H, W, w2.shape[0] - 1), float("nan"))
    conf = torch.full((Fr, H, W), float("nan"))
    bias32, w232, b232 = bias.float(), w2.float(), b2.float()
    stages = [torch.zeros(130, 128), torch.zeros(130, 128)]
    st = 0
    moved = None
    for item in range(sch["n_items"]):
        seg, strip = item % sch["n_segs"], (item // sch["n_segs"]) % sch["n_strips"]
        f = item // (sch["n_segs"] * sch["n_strips"])
        ya = seg * sch["seg_rows"]
        yb = min(ya + sch["seg_rows"], H)
        x0 = 128 * strip
        x_lo, x_hi, xs_lo, ns, itab = R.tail_strip(w, W, strip)
        if mistake == "itab" and moved is None and ns > 4:
            j = ns // 2
            (r0a, na), (r0b, nb) = itab[j - 1], itab[j]
            itab[j - 1], itab[j] = (r0a, na + 1), (r0b + 1, nb - 1)
            moved = x0 - 1 + r0b
        pairs = [(row0 + k, j) for j, (row0, n) in enumerate(itab) for k in range(n)]
        assert sorted(r for r, _ in pairs) == list(range(x_lo - (x0 - 1), x_hi - (x0 - 1) + 1))    # every pixel exactly once
        rows = torch.tensor([r for r, _ in pairs])
        js = torch.tensor([j for _, j in pairs])
        Xs = (x0 - 1 + rows).numpy().astype(np.float32)
        wx1 = torch.from_numpy((sx * Xs) - (xs_lo + js.numpy()).astype(np.float32))
        wx0 = 1.0 - wx1
        zrow = W - x0 + 1
        p1 = torch.zeros(128, 32)
        p2 = torch.zeros(128, 32)
        for r in range(ya - 1 if mistake != "halo" or ya == 0 else ya, yb + 1):
            if 0 <= r < H:
                fy = sy * np.float32(r)
                y0 = int(fy)
                y1 = y0 + (1 if y0 < h - 1 else 0)
                wy1 = torch.tensor(fy - np.float32(y0))
                wy0 = 1.0 - wy1
                v0 = src32[f, y0, xs_lo:xs_lo + ns]
                v1 = src32[f, y1, xs_lo:xs_lo + ns]
                vert = _fma(wy1, v1, wy0 * v0)                                   # ffma2(wy1, v1, fmul2(wy0, v0))
                A = stages[st]
                if x0 == 0:
                    A[0] = 0
                if zrow < 130 and mistake != "zero_col":
                    A[zrow] = 0
                va, vb = vert[js], vert[(js + 1).clamp(max=ns - 1)]
                A[rows] = _store16(_fma(wx1[:, None], vb, wx0[:, None] * va), dtype)
                st ^= 1
                d = torch.cat([A[0:128], A[1:129], A[2:130]], 1) @ wcat         # [128, 96]: ky = 2 | 1 | 0
            else:
                d = torch.zeros(128, 96)
            d2 = d[:, :32] + p1
            p1 = p2 + d[:, 32:64]
            p2 = d[:, 64:]
            y = r - 1
            if not (ya <= y < yb):
                continue
            X = torch.arange(x0, x0 + 128)
            keep = X < W
            X = X[keep]
            v = d2[keep] + bias32
            if gx is not None:
                xcls = torch.where(X == 0, 0, torch.where(X == W - 1, 2, 1))
                ycls = 0 if y == 0 else (2 if y == H - 1 else 1)
                if mistake == "row_class":
                    ycls = 1
                v = v + (gy[xcls, y] + gx[ycls, X])
            a = torch.relu(v) @ w232.t() + b232
            ap = a[:, :-1]
            preds[f, y, X] = torch.exp(ap) if head_act == 0 else torch.sign(ap) * torch.expm1(ap.abs())
            conf[f, y, X] = torch.exp(a[:, -1]) if mistake == "conf" else 1.0 + torch.exp(a[:, -1])
    return preds, conf, moved


def _tail_case(dtype, h=24, w=296, H=41, W=518, outc=4, seed=0, tables=True):
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(1, h, w, 128, generator=g, dtype=F64).to(dtype).to(F64)
    wb = (torch.randn(32, 9 * 128, generator=g, dtype=F64) * (9 * 128) ** -0.5).to(dtype).to(F64)
    b1 = (torch.randn(32, generator=g) * 0.1).double()
    w2 = (torch.randn(outc, 32, generator=g) * 32 ** -0.5).double()
    b2 = (torch.randn(outc, generator=g) * 0.1).double()
    tx = torch.randn(W, 64, generator=g) * 0.1 if tables else None
    ty = torch.randn(H, 64, generator=g) * 0.1 if tables else None
    return src, tx, ty, wb, b1, w2, b2, H, W


@pytest.fixture(scope="module")
def tail_refs():
    out = {}
    for dtype in (BF16, F16):
        case = _tail_case(dtype)
        src, tx, ty, wb, b1, w2, b2, H, W = case
        out[dtype] = case, R.dpt_tail_ref(src, tx, ty, wb, b1, w2, b2, 1, H, W, dtype)
    return out


def _tail_checks(preds, conf, ref):
    rp, rc, bp, bc = ref
    return [lambda: R.check_bound(preds, rp, bp, "tail preds", ("frame", "y", "x", "c")),
            lambda: R.check_bound(conf, rc, bc, "tail conf", ("frame", "y", "x"))]


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_tail_emulation_passes_bound(dtype, tail_refs):
    """296 -> 518 wide (five strips, the last one 6 pixels), 24 -> 41 rows in segments of 8 with their halo rows."""
    (src, tx, ty, wb, b1, w2, b2, H, W), ref = tail_refs[dtype]
    sch = R.tail_schedule(1, H, W, 132)
    assert sch["n_strips"] == 5 and sch["n_segs"] > 1
    preds, conf, _ = _emulate_tail(src, tx, ty, wb, b1, w2, b2, 1, H, W, dtype)
    rp, rc, bp, bc = ref
    r1 = R.check_bound(preds, rp, bp, "emulated tail preds", ("frame", "y", "x", "c"))
    r2 = R.check_bound(conf, rc, bc, "emulated tail conf", ("frame", "y", "x"))
    assert max(r1, r2) < 0.75, (r1, r2)


@pytest.mark.parametrize("mistake", ["halo", "zero_col", "row_class", "itab", "conf"])
def test_tail_seeded_mistakes_fail(mistake, tail_refs):
    (src, tx, ty, wb, b1, w2, b2, H, W), ref = tail_refs[BF16]
    preds, conf, moved = _emulate_tail(src, tx, ty, wb, b1, w2, b2, 1, H, W, BF16, mistake=mistake)
    msg = _failure(_tail_checks(preds, conf, ref))
    assert msg is not None, f"{mistake} passed the bound"
    sch = R.tail_schedule(1, H, W, 132)
    if mistake == "halo":
        assert _at(msg, "y") in range(sch["seg_rows"], H, sch["seg_rows"]), msg
    elif mistake == "zero_col":
        assert _at(msg, "x") == W - 1, msg
    elif mistake == "row_class":
        assert _at(msg, "y") in (0, H - 1), msg
    elif mistake == "itab":
        assert moved is not None and abs(_at(msg, "x") - moved) <= 1, (msg, moved)
    else:
        assert msg.startswith("tail conf"), msg


def test_tail_tables_compose_to_the_embedding_conv():
    """gx[rc(y), x] + gy[cc(x), y] is the 3x3 convolution of the embedding map, border classes included."""
    g = torch.Generator().manual_seed(3)
    H, W = 6, 9
    tx, ty = torch.randn(W, 64, generator=g), torch.randn(H, 64, generator=g)
    wb = torch.randn(32, 9 * 128, generator=g).double()
    gx, gy = R.tail_tables_ref(tx, ty, wb, H, W)
    cls = lambda n: torch.tensor([0] + [1] * (n - 2) + [2])                        # noqa: E731
    comp = gx[cls(H)] + gy[cls(W)].permute(1, 0, 2)
    conv = R.conv3x3(R.embedding_map(tx, ty, H, W, 128)[None], wb.reshape(32, 3, 3, 128))[0]
    assert torch.allclose(comp, conv, rtol=0, atol=1e-12)
    # the interior class on a border row is a different table
    assert not torch.allclose(gx[1], gx[0]) and not torch.allclose(gy[1], gy[2])


# ----------------------------------------------------------------------------------------------- upsampling
def _emulate_upsample(src, H, W, tx, ty, dtype, mistake=None):
    """upsample_rows_kernel in fp32: vertical blend of two source rows into a shared row, horizontal blend out of it, + table,
    16-bit store.  The shared row holds w pixels; what lies past it reads as NaN (uninitialised shared memory).  Mistakes:
    "align_corners_false" (s = h / H), "x1_unclamped" (x1 = x0 + 1 at the last column), "swap_wy" (wy0 and wy1 swapped)."""
    Fr, h, w, C = src.shape

    def pos(n, N, x_axis=False):
        s = np.float32(n) / np.float32(N) if mistake == "align_corners_false" else np.float32(n - 1) / np.float32(N - 1)
        f = s * np.arange(N, dtype=np.float32)
        i0 = f.astype(np.int64)
        i1 = i0 + 1 if (mistake == "x1_unclamped" and x_axis) else i0 + (i0 < n - 1)
        w1 = f - i0.astype(np.float32)
        return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(1 - w1), torch.from_numpy(w1)
    yi0, yi1, wy0, wy1 = pos(h, H)
    if mistake == "swap_wy":
        wy0, wy1 = wy1, wy0
    xi0, xi1, wx0, wx1 = pos(w, W, x_axis=True)
    s = src.float()
    row = wy0[None, :, None, None] * s[:, yi0] + wy1[None, :, None, None] * s[:, yi1]             # [F, H, w, C]
    row = torch.cat([row, torch.full_like(row[:, :, :1], float("nan"))], 2)
    out = wx0[None, None, :, None] * row[:, :, xi0] + wx1[None, None, :, None] * row[:, :, xi1]
    if tx is not None:
        out = out + R.embedding_map(tx, ty, H, W, C).float()[None]
    return _store16(out, dtype)


@pytest.mark.parametrize("mistake", [None, "align_corners_false", "x1_unclamped", "swap_wy"])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_upsample_emulation_and_seeded_mistakes(mistake, dtype):
    """19 -> 37 (s = 1/2: the last column samples x0 = w - 1 exactly) and 8 x 12 -> 14 x 21, with tables."""
    for (h, w, H, W) in ((19, 19, 37, 37), (8, 12, 14, 21)):
        g = torch.Generator().manual_seed(h)
        C = 64
        src = torch.randn(2, h, w, C, generator=g, dtype=F64).to(dtype).to(F64)
        tx, ty = torch.randn(W, C // 2, generator=g) * 0.1, torch.randn(H, C // 2, generator=g) * 0.1
        ref, bound = R.bilinear_ref(src, H, W, tx, ty, dtype)
        out = _emulate_upsample(src, H, W, tx, ty, dtype, mistake)
        if mistake is None:
            r, f = R.check_rounded(out, ref, bound, dtype, "emulated upsample", ("frame", "y", "x", "c"))
            assert r < 0.75 and f > 0.995, (r, f)
        elif mistake == "x1_unclamped" and (w - 1) / (W - 1) != 0.5:
            continue                      # the last column lands at x0 = w - 1 only where fp32(s (W - 1)) reaches w - 1
        else:
            with pytest.raises(AssertionError):
                R.check_rounded(out, ref, bound, dtype, f"upsample with {mistake}", ("frame", "y", "x", "c"))


def test_upsample_path_rule():
    assert R.upsample_path(296, 256) == "rows" and R.upsample_path(384, 128) == "rows"
    assert R.upsample_path(385, 128) == "direct" and R.upsample_path(12, 48) == "direct" and R.upsample_path(19, 144) == "direct"


def test_sample_positions_are_the_kernels_fp32_steps():
    """w1 = f - i0 is exact, i1 clamps at the last source pixel, and a non-dyadic scale puts f a few fp32 ulps off s o."""
    i0, i1, w0, w1, f = R.sample_positions(296, 518)
    assert int(i1.max()) == 295 and int(i0.max()) <= 295
    assert torch.equal(w1, f - i0.double()) and bool(((w0 + w1) - 1).abs().max() <= 2 ** -24)
    exact = torch.arange(518, dtype=F64) * 295 / 517
    assert 0 < float((f - exact).abs().max()) < 1e-4


# ----------------------------------------------------------------------------------------------- geometry pin
def test_tail_geometry_pin():
    """For every (w, W) with 2 <= w < 400, W < 1100 that ovg_dpt_tail_supported accepts, restated in fp32: every strip spans at
    most FT_VBUF_PX = 80 source pixels (the ring row and the itab size), and the producers' interval runs (start at
    int(s / sx) - 2, walk up while int(sx X) < s, count while == s) cover [x_lo, x_hi] exactly once."""
    f32 = np.float32
    accepted = span80 = 0
    for w in range(2, 400):
        Wv = np.arange(w, 1100)
        sx = f32(w - 1) / (Wv - 1).astype(f32)
        span = (sx * f32(129.0)).astype(np.int64) + 3
        ok = span <= R.FT_VBUF_PX
        Wv, sx = Wv[ok], sx[ok]
        accepted += len(Wv)
        span80 += int((span[ok] == R.FT_VBUF_PX).sum())
        nstrips = (Wv + 127) // 128
        for strip in range(int(nstrips.max(initial=0))):
            sel = nstrips > strip
            Ws, s = Wv[sel], sx[sel]
            x0 = 128 * strip
            x_lo = max(x0 - 1, 0)
            x_hi = np.minimum(x0 + 128, Ws - 1)
            xs_lo = (s * f32(x_lo)).astype(np.int64)
            xs_hi = np.minimum((s * x_hi.astype(f32)).astype(np.int64) + 1, w - 1)
            ns = xs_hi - xs_lo + 1
            assert (ns <= R.FT_VBUF_PX).all(), (w, Ws[ns > R.FT_VBUF_PX][:4], strip)
            X = x_lo + np.arange(130)[None, :]
            valid = X <= x_hi[:, None]
            sX = (s[:, None] * X.astype(f32)).astype(np.int64)
            j = sX - xs_lo[:, None]
            assert (~valid | ((j >= 0) & (j < ns[:, None]))).all(), (w, strip)
            start = np.maximum((sX.astype(f32) / s[:, None]).astype(np.int64) - 2, x_lo)
            assert (~valid | (start <= X)).all(), (w, strip)
    print(f"{accepted} accepted geometries, {span80} with span 80")
    assert accepted > 200000 and span80 > 300
    # the scalar walk (used by the emulation) agrees on a few of them
    for w, W in ((296, 518), (49, 385), (224, 392), (370, 641), (220, 383)):
        for strip in range((W + 127) // 128):
            x_lo, x_hi, _, ns, itab = R.tail_strip(w, W, strip)
            assert ns <= R.FT_VBUF_PX and sum(n for _, n in itab) == x_hi - x_lo + 1
