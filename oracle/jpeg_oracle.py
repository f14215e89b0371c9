"""CPU restatement of baseline JPEG decoding as Pillow runs it (libjpeg-turbo defaults)  --  TEST INFRASTRUCTURE.

Every step the device decoder (csrc/jpeg.cuh) reproduces, in numpy / pure Python, citing the libjpeg-turbo function it restates:

* ``parse``: the marker walk (jdmarker.c get_sof / get_sos / get_dht / get_dqt / get_dri, jdapimin.c default_decompress_parms for
  the colour space), the routing decision (device or Pillow, and why) and the unstuffed restart segments.
* ``huffman_decode``: serial decode of one scan (jdhuff.c jpeg_make_d_derived_tbl, decode_mcu, HUFF_EXTEND), DC prediction reset
  at every restart marker (process_restart).
* ``idct_islow``: jidctint.c jpeg_idct_islow, CONST_BITS 13, PASS1_BITS 2, dequantisation inside, and the masked post-IDCT range
  limit of jdmaster.c prepare_range_limit_table (``& 1023``).  That is the C code; on x86-64 Pillow's libjpeg-turbo runs the SIMD
  islow instead (16-bit dequantisation and pairwise sums, pass-1 outputs saturated to int16, final samples clamped).  The two agree
  only while dequantised coefficients and pass-1 outputs stay within +-16383 and the samples before the range limit within
  [-512, 511]; ``idct_islow`` raises outside that range, where the device flags the file for Pillow.
* ``upsample``: jdsample.c h2v1_fancy_upsample / h2v2_fancy_upsample (edge rows repeated as jdmainct.c does), and the plain
  replicating upsamplers libjpeg-turbo picks when the downsampled width is 2 or less.
* ``ycc_to_rgb``: jdcolor.c build_ycc_rgb_table / ycc_rgb_convert (SCALEBITS 16).

tests/test_jpeg.py checks ``decode`` against ``np.asarray(Image.open(p).convert("RGB"))`` bit for bit, and the library's plan
against ``parse``.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Tuple

import numpy as np

# routing reasons: the values of OVG_JPEG_* in include/ovg.h
DEVICE, NOT_JPEG, TRUNCATED, PROCESS, PRECISION, COLOR, SAMPLING, SCANS, TABLES, MARKER, RESTART, SIZE = range(12)
REASONS = ("device", "not a JPEG", "truncated", "not baseline / extended Huffman", "not 8-bit", "colour space", "sampling",
           "several scans or partial scan", "missing or invalid table", "unexpected marker", "restart markers", "size")

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                   61, 54, 47, 55, 62, 63], np.int64)     # jutils.c jpeg_natural_order


@dataclass
class Parsed:
    route: int = DEVICE
    width: int = 0
    height: int = 0
    comps: List[Tuple[int, int, int, int]] = field(default_factory=list)     # (id, h, v, quant table) in frame order
    tables: List[Tuple[int, int]] = field(default_factory=list)              # (dc, ac) Huffman table per component
    quant: Dict[int, np.ndarray] = field(default_factory=dict)               # table -> 64 values in natural order
    huff: Dict[Tuple[int, int], Tuple[List[int], List[int]]] = field(default_factory=dict)   # (class, id) -> (bits[16], vals)
    restart: int = 0
    segments: List[bytes] = field(default_factory=list)

    @property
    def gray(self) -> bool:
        return len(self.comps) == 1

    @property
    def mcu_geometry(self):
        """(hmax, vmax, MCUs per row, MCU rows); one component: one block per MCU (non-interleaved scan, jdinput.c)."""
        if self.gray:
            return 1, 1, -(-self.width // 8), -(-self.height // 8)
        hm, vm = max(c[1] for c in self.comps), max(c[2] for c in self.comps)
        return hm, vm, -(-self.width // (8 * hm)), -(-self.height // (8 * vm))


def _be16(d: bytes, i: int) -> int:
    return (d[i] << 8) | d[i + 1]


def _valid_huff(bits, vals, is_dc) -> bool:
    """jdhuff.c jpeg_make_d_derived_tbl: the code lengths must fit, DC symbols must be <= 15."""
    code, k = 0, 0
    for l in range(1, 17):
        code += bits[l - 1]
        if code >= (1 << l):                               # no code may be all ones
            return False
        code <<= 1
    return sum(bits) <= 256 and (not is_dc or all(v <= 15 for v in vals))


def unstuff(d: bytes, i: int):
    """Entropy-coded bytes from i to the first marker other than RST: (segments, RST numbers seen, index of that marker).
    FF 00 is a data byte FF; FF D0..D7 end a restart segment.  Returns None at a fill byte run (FF FF) inside the data."""
    segs, rsts, cur = [], [], bytearray()
    n = len(d)
    while True:
        j = d.find(b"\xff", i)
        if j < 0 or j + 1 >= n:
            return None
        cur += d[i:j]
        m = d[j + 1]
        if m == 0:
            cur.append(0xFF)
            i = j + 2
        elif 0xD0 <= m <= 0xD7:
            segs.append(bytes(cur))
            rsts.append(m - 0xD0)
            cur = bytearray()
            i = j + 2
        elif m == 0xFF:
            return None
        else:
            segs.append(bytes(cur))
            return segs, rsts, j


def parse(d: bytes) -> Parsed:
    p = Parsed()

    def out(r):
        p.route = r
        return p
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        return out(NOT_JPEG)
    i, n = 2, len(d)
    jfif = adobe = False
    transform = -1
    sof = False
    while True:
        if i + 4 > n:
            return out(TRUNCATED)
        if d[i] != 0xFF:
            return out(MARKER)
        while i < n and d[i] == 0xFF:
            i += 1
        if i + 3 > n:
            return out(TRUNCATED)
        m = d[i]
        i += 1
        if m == 0xD9 or 0xD0 <= m <= 0xD7 or m == 0x01:
            return out(MARKER if m != 0xD9 else SCANS)
        ln = _be16(d, i)
        if ln < 2 or i + ln > n:
            return out(TRUNCATED)
        seg = d[i + 2:i + ln]
        if m == 0xE0 and len(seg) >= 14 and seg[:5] == b"JFIF\x00":      # jdmarker.c examine_app0 (APP0_DATA_LEN)
            jfif = True
        elif m == 0xEE and len(seg) >= 12 and seg[:5] == b"Adobe":       # jdmarker.c examine_app14
            adobe, transform = True, seg[11]
        elif 0xE0 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDB:                                                  # get_dqt
            k = 0
            while k < len(seg):
                pq, tq = seg[k] >> 4, seg[k] & 15
                sz = 128 if pq else 64
                if tq > 3 or k + 1 + sz > len(seg):
                    return out(TABLES)
                raw = np.frombuffer(seg[k + 1:k + 1 + sz], ">u2" if pq else np.uint8).astype(np.int64)
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = raw
                p.quant[tq] = q
                k += 1 + sz
        elif m == 0xC4:                                                  # get_dht
            k = 0
            while k < len(seg):
                if k + 17 > len(seg):
                    return out(TABLES)
                tc, th = seg[k] >> 4, seg[k] & 15
                bits = list(seg[k + 1:k + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or cnt > 256 or k + 17 + cnt > len(seg):
                    return out(TABLES)
                p.huff[(tc, th)] = (bits, list(seg[k + 17:k + 17 + cnt]))
                k += 17 + cnt
        elif m == 0xDD:                                                  # get_dri
            if ln != 4:
                return out(MARKER)
            p.restart = _be16(seg, 0)
        elif 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):        # get_sof
            if sof:
                return out(MARKER)
            sof = True
            if m not in (0xC0, 0xC1):
                return out(PROCESS)
            if len(seg) < 6:
                return out(MARKER)
            if seg[0] != 8:
                return out(PRECISION)
            p.height, p.width, nc = _be16(seg, 1), _be16(seg, 3), seg[5]
            if len(seg) != 6 + 3 * nc:
                return out(MARKER)
            p.comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(nc)]
        elif m == 0xDA:                                                  # get_sos
            if not sof:
                return out(MARKER)
            if p.height == 0 or p.width == 0:
                return out(SIZE)
            nc = len(p.comps)
            if nc == 3:                                                  # jdapimin.c default_decompress_parms
                ids = tuple(c[0] for c in p.comps)
                if not jfif and adobe and transform == 0:
                    return out(COLOR)
                if not jfif and not adobe and ids in ((82, 71, 66), (1, 0x22, 0x23)):
                    return out(COLOR)
                (_, h0, v0, _), c1, c2 = p.comps
                if (h0, v0) not in ((1, 1), (2, 1), (2, 2)) or c1[1:3] != (1, 1) or c2[1:3] != (1, 1):
                    return out(SAMPLING)
            elif nc == 1:
                if not 1 <= p.comps[0][1] <= 4 or not 1 <= p.comps[0][2] <= 4:
                    return out(SAMPLING)
            else:
                return out(COLOR)
            ns = seg[0]
            if ns != nc or len(seg) != 4 + 2 * ns:
                return out(SCANS)
            if tuple(seg[1 + 2 * c] for c in range(ns)) != tuple(c[0] for c in p.comps):
                return out(SCANS)
            if tuple(seg[1 + 2 * ns:4 + 2 * ns]) != (0, 63, 0):
                return out(SCANS)
            p.tables = [(seg[2 + 2 * c] >> 4, seg[2 + 2 * c] & 15) for c in range(ns)]
            for (dc, ac), comp in zip(p.tables, p.comps):
                if comp[3] not in p.quant or (0, dc) not in p.huff or (1, ac) not in p.huff:
                    return out(TABLES)
                if not _valid_huff(*p.huff[(0, dc)], True) or not _valid_huff(*p.huff[(1, ac)], False):
                    return out(TABLES)
            r = unstuff(d, i + ln)
            if r is None:
                return out(TRUNCATED)
            segs, rsts, j = r
            if d[j + 1] != 0xD9:
                return out(SCANS if d[j + 1] in (0xDA, 0xDC) or 0xC0 <= d[j + 1] <= 0xFE else MARKER)
            _, _, mx, my = p.mcu_geometry
            nmcu = mx * my
            want = -(-nmcu // p.restart) if p.restart else 1
            if len(segs) != want or rsts != [k % 8 for k in range(want - 1)]:
                return out(RESTART)
            p.segments = segs
            return p
        else:
            return out(MARKER)
        i += ln


class _Table:
    """jdhuff.c jpeg_make_d_derived_tbl: a 16-bit lookahead (length, symbol) table."""

    def __init__(self, bits, vals):
        self.length = np.zeros(1 << 16, np.int64)
        self.symbol = np.zeros(1 << 16, np.int64)
        code, k = 0, 0
        for l in range(1, 17):
            for _ in range(bits[l - 1]):
                lo = code << (16 - l)
                self.length[lo:lo + (1 << (16 - l))] = l
                self.symbol[lo:lo + (1 << (16 - l))] = vals[k]
                code, k = code + 1, k + 1
            code <<= 1
        self.length, self.symbol = self.length.tolist(), self.symbol.tolist()


def _extend(v: int, s: int) -> int:
    return v - (1 << s) + 1 if v < (1 << (s - 1)) else v       # HUFF_EXTEND


def huffman_decode(p: Parsed) -> List[np.ndarray]:
    """Coefficients per component [blocks_y, blocks_x, 64] (natural order, DC absolute, int16 as JCOEF stores them).
    Raises ValueError where libjpeg-turbo would warn (code not in the table, a coefficient past z = 63, too little data):
    the device flags exactly those files."""
    hm, vm, mx, my = p.mcu_geometry
    samp = [(1, 1)] if p.gray else [(c[1], c[2]) for c in p.comps]
    coefs = [np.zeros((my * v, mx * h, 64), np.int64) for h, v in samp]
    dc_t = [_Table(*p.huff[(0, t[0])]) for t in p.tables]
    ac_t = [_Table(*p.huff[(1, t[1])]) for t in p.tables]
    nmcu = mx * my
    per_seg = p.restart or nmcu
    for si, seg in enumerate(p.segments):
        nbits = 8 * len(seg)
        bits = (bin(int.from_bytes(b"\x01" + seg, "big"))[3:] if seg else "") + "0" * 64
        pos = 0
        last = [0] * len(samp)                                # process_restart: DC predictions reset
        for m in range(si * per_seg, min(nmcu, (si + 1) * per_seg)):
            by0, bx0 = divmod(m, mx)
            for c, (h, v) in enumerate(samp):
                for sub in range(h * v):
                    blk = coefs[c][by0 * v + sub // h, bx0 * h + sub % h]
                    look = int(bits[pos:pos + 16], 2)
                    l = dc_t[c].length[look]
                    if l == 0:
                        raise ValueError("code not in the DC table")
                    s = dc_t[c].symbol[look]
                    pos += l
                    diff = _extend(int(bits[pos:pos + s], 2), s) if s else 0
                    pos += s
                    last[c] += diff
                    blk[0] = np.int16(np.int64(last[c]).astype(np.int16))
                    k = 1
                    while k < 64:
                        look = int(bits[pos:pos + 16], 2)
                        l = ac_t[c].length[look]
                        if l == 0:
                            raise ValueError("code not in the AC table")
                        rs = ac_t[c].symbol[look]
                        pos += l
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            if k > 63:
                                raise ValueError("coefficient past z = 63")
                            blk[ZIGZAG[k]] = _extend(int(bits[pos:pos + s], 2), s)
                            pos += s
                        else:
                            if r != 15:
                                break
                            k += 15
                            if k > 63:
                                raise ValueError("zero run past z = 63")
                        k += 1
                    if pos > nbits:
                        raise ValueError("segment ends early")
    return [c.astype(np.int16) for c in coefs]


FIX = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137, f1961=16069,
           f2053=16819, f2562=20995, f3072=25172)


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7, shift):
    """One pass of jidctint.c jpeg_idct_islow over arrays (int64); returns the 8 outputs DESCALEd by `shift`."""
    F = FIX
    z2, z3 = x2, x6
    z1 = (z2 + z3) * F["f0541"]
    tmp2 = z1 + z3 * -F["f1847"]
    tmp3 = z1 + z2 * F["f0765"]
    tmp0 = (x0 + x4) << 13
    tmp1 = (x0 - x4) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = x7, x5, x3, x1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F["f1175"]
    t0, t1, t2, t3 = t0 * F["f0298"], t1 * F["f2053"], t2 * F["f3072"], t3 * F["f1501"]
    z1, z2, z3, z4 = z1 * -F["f0899"], z2 * -F["f2562"], z3 * -F["f1961"], z4 * -F["f0390"]
    z3, z4 = z3 + z5, z4 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    r = 1 << (shift - 1)
    return [(tmp10 + t3 + r) >> shift, (tmp11 + t2 + r) >> shift, (tmp12 + t1 + r) >> shift, (tmp13 + t0 + r) >> shift,
            (tmp13 - t0 + r) >> shift, (tmp12 - t1 + r) >> shift, (tmp11 - t2 + r) >> shift, (tmp10 - t3 + r) >> shift]


IDCT_IN_MAX, IDCT_OUT_MIN, IDCT_OUT_MAX = 16383, -512, 511


def range_limit(x: np.ndarray) -> np.ndarray:
    """idct_table[x & RANGE_MASK] of jdmaster.c prepare_range_limit_table: x + 128 clamped on [-512, 511], periodic in 1024."""
    v = x & 1023
    return np.where(v < 128, v + 128, np.where(v < 512, 255, np.where(v < 896, 0, v - 896))).astype(np.uint8)


def idct_islow(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """coef [..., 64] int16 natural order, q [64] -> samples [..., 8, 8] uint8 (jpeg_idct_islow).  Raises ValueError for a
    block outside the range where libjpeg-turbo's C and SIMD IDCTs agree (see the module docstring)."""
    c = (coef.astype(np.int64) * q.astype(np.int64)).reshape(coef.shape[:-1] + (8, 8))
    cols = _idct_1d(*[c[..., k, :] for k in range(8)], 13 - 2)                       # pass 1: columns, keep PASS1_BITS
    ws = np.stack(cols, -2)
    rows = np.stack(_idct_1d(*[ws[..., :, k] for k in range(8)], 13 + 2 + 3), -1)    # pass 2: rows
    if (np.abs(c) > IDCT_IN_MAX).any() or (np.abs(ws) > IDCT_IN_MAX).any() or \
            (rows < IDCT_OUT_MIN).any() or (rows > IDCT_OUT_MAX).any():
        raise ValueError("IDCT outside the range where libjpeg-turbo's C and SIMD paths agree")
    return range_limit(rows)


def planes(p: Parsed, coefs) -> List[np.ndarray]:
    qs = [p.quant[c[3]] for c in p.comps]
    out = []
    for cf, q in zip(coefs, qs):
        s = idct_islow(cf, q)                                   # [by, bx, 8, 8]
        out.append(s.transpose(0, 2, 1, 3).reshape(s.shape[0] * 8, s.shape[1] * 8))
    return out


def upsample(c: np.ndarray, dw: int, dh: int, h2: int, v2: int) -> np.ndarray:
    """Chroma plane [>= dh, >= dw] (block padded) to [dh * v2, dw * h2] int64 (jdsample.c)."""
    c = c.astype(np.int64)
    if h2 == 1:
        return c[:dh, :dw]
    if dw <= 2:                                              # jinit_upsampler: no fancy upsampling for widths of 2 or less
        return np.repeat(np.repeat(c[:dh], 2, 1), v2, 0)[:, :2 * dw]
    k = np.arange(dw)
    prv, nxt = np.maximum(k - 1, 0), np.minimum(k + 1, dw - 1)
    if v2 == 1:                                              # h2v1_fancy_upsample
        x = c[:dh]
        o = np.empty((dh, 2 * dw), np.int64)
        o[:, 0::2] = (3 * x[:, k] + x[:, prv] + 1) >> 2
        o[:, 1::2] = (3 * x[:, k] + x[:, nxt] + 2) >> 2
        o[:, 0], o[:, -1] = x[:, 0], x[:, dw - 1]
        return o
    r = np.arange(dh)
    o = np.empty((2 * dh, 2 * dw), np.int64)
    for v, nb in ((0, np.maximum(r - 1, 0)), (1, np.minimum(r + 1, dh - 1))):   # h2v2_fancy_upsample, edge rows repeated
        s = 3 * c[r][:, :dw] + c[nb][:, :dw]
        e = (3 * s[:, k] + s[:, prv] + 8) >> 4
        f = (3 * s[:, k] + s[:, nxt] + 7) >> 4
        e[:, 0] = (4 * s[:, 0] + 8) >> 4
        f[:, -1] = (4 * s[:, dw - 1] + 7) >> 4
        o[v::2, 0::2], o[v::2, 1::2] = e, f
    return o


def ycc_to_rgb(y, cb, cr) -> np.ndarray:
    """jdcolor.c build_ycc_rgb_table + ycc_rgb_convert (SCALEBITS 16, ONE_HALF 1 << 15, range_limit clamps)."""
    def fix(x):
        return int(x * 65536 + 0.5)
    x = np.arange(256, dtype=np.int64) - 128
    cr_r = (fix(1.40200) * x + (1 << 15)) >> 16
    cb_b = (fix(1.77200) * x + (1 << 15)) >> 16
    cr_g = -fix(0.71414) * x
    cb_g = -fix(0.34414) * x + (1 << 15)
    y = y.astype(np.int64)
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> 16)
    b = y + cb_b[cb]
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data: bytes) -> np.ndarray:
    """uint8 RGB [h, w, 3] of a device-routed JPEG, as Pillow's Image.open(...).convert("RGB") gives it."""
    p = parse(data)
    if p.route != DEVICE:
        raise ValueError(f"not device-decodable: {REASONS[p.route]}")
    pl = planes(p, huffman_decode(p))
    W, H = p.width, p.height
    if p.gray:
        y = pl[0][:H, :W]
        return np.repeat(y[..., None], 3, -1)
    hm, vm, _, _ = p.mcu_geometry
    dw, dh = -(-W // hm), -(-H // vm)                        # chroma downsampled size (jdmaster.c)
    cb = upsample(pl[1], dw, dh, hm, vm)[:H, :W]
    cr = upsample(pl[2], dw, dh, hm, vm)[:H, :W]
    return ycc_to_rgb(pl[0][:H, :W], cb, cr)


# ---------------------------------------------------------------------------------------------------------------- fixtures
def octave_noise(width: int, height: int, seed: int = 0) -> np.ndarray:
    """uint8 RGB [h, w, 3]: a sum of bicubically upscaled seeded noise at several scales.  Camera-like entropy: about 2.2 bits
    per pixel at quality 90 4:2:0 and 4.3 at quality 95 4:2:2 (smooth upscaled images give well under 1)."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    acc = np.zeros((height, width, 3), np.float32)
    for f, wgt in ((64, 0.4), (16, 0.3), (4, 0.18), (2, 0.08), (1, 0.04)):
        small = rng.integers(0, 256, (max(1, height // f), max(1, width // f), 3), dtype=np.uint8)
        big = small if f == 1 else np.asarray(Image.fromarray(small).resize((width, height), Image.Resampling.BICUBIC))
        acc += wgt * big.astype(np.float32)
    return np.clip(acc + 0.5, 0, 255).astype(np.uint8)


def encode(rgb: np.ndarray, gray: bool = False, **kw) -> bytes:
    """Pillow's JPEG encoding of an RGB array (grayscale: converted to "L" first)."""
    import io
    from PIL import Image
    im = Image.fromarray(rgb)
    if gray:
        im = im.convert("L")
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()
