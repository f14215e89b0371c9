"""The post-processing kernels that run right after the forward, element by element.

- percentile_f32, the oracle's restatement of numpy >= 2's percentile, against np.percentile itself (CPU);
- ovg_conf_percentile_mask against it to the bit: threshold, mask and kept count, over sizes that take every tail and
  grid-stride path, ties, signed zeros, subnormals, infinities at and next to the selected ranks, and NaN;
- the point cloud's centre (fsum) and scale (its 5th / 95th percentiles to the bit, the norm to 1 ulp);
- ovg_pose_decode and ovg_unproject_depth per element against the same formulas in fp64, with bounds derived from each
  element's operation count (never scaled by the largest element), on outputs filled with NaN so an unwritten element fails.
"""
import math
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle.postprocess_oracle import percentile_f32

F32 = np.float32
U = 2.0 ** -24                 # unit roundoff of fp32
ETA = 2.0 ** -149              # smallest subnormal: the absolute error an fp32 result can lose to gradual underflow

NUMPY2 = int(np.__version__.split(".")[0]) >= 2
needs_numpy2 = pytest.mark.skipif(not NUMPY2, reason="percentile_f32 restates numpy >= 2's fp32 rule (NEP 50); "
                                                     f"numpy {np.__version__} interpolates in fp64")

VIEWS8, VIEWS24 = 8 * 518 * 518, 24 * 518 * 518           # 2,146,592 and 6,439,776 confidences
SIZES = (1, 2, 3, 4, 5, 7, 8, 9, 1001, 2 ** 24 - 1, 2 ** 24 + 1, 2 ** 24 + 2, 2 ** 24 + 3, VIEWS8, VIEWS24)
PCTS = (0.0, 100.0, 50.0, 25.0, 12.5, 37.3, 99.9, 1e-7, 100 - 1e-5, 66.6)
NANS = (0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFC12345)   # quiet +/-, signalling, negative with a payload


def _ranks(n, p):
    """The two ranks numpy's rule selects (to place infinities at and next to them).  Above 2^24 the upper one is the fp32
    sum floor(vi) + 1, which rounds to even."""
    last = F32(n - 1)
    vi = last * (F32(p) / F32(100))
    if vi >= last:
        return n - 1, n - 1
    r = int(np.floor(vi))
    return r, min(int(F32(r) + F32(1)), n - 1)


@lru_cache(maxsize=2)
def _base(n):
    """Confidence-like values of both signs over many magnitudes: ties, -0 / +0, subnormals and negatives included."""
    rng = np.random.default_rng(n)
    a = (rng.standard_normal(n) * np.exp(2 * rng.standard_normal(n))).astype(F32)
    a[::7] = a[0]
    special = np.array([-0.0, 0.0, 1e-40, -1e-42, 1.4e-45, -3.0, 0.1], F32)
    k = min(n, special.size)
    at = rng.permutation(n)[:k]
    a[at] = special[:k]
    return a


def _with_infs(a, p, kind, seed, is_sorted=False):
    """a with -inf / +inf on the low / high side of the selected ranks: on them ("at") or just beside them ("next");
    "huge_at": -3e38 up to the lower rank and +3e38 from the upper one, so hi - lo overflows to +inf."""
    n = a.size
    r0, r1 = _ranks(n, p)
    # ranks r0 and r1 in place, smaller values before, larger after
    s = a.copy() if is_sorted else np.partition(a, sorted({r0, r1}))
    lo_end, hi_start = (r0 + 1, r1) if kind.endswith("at") else (r0, r1 + 1)
    if kind.startswith(("lo", "both", "huge")):
        s[:lo_end] = -3e38 if kind.startswith("huge") else -np.inf
    if kind.startswith(("hi", "both", "huge")):
        s[hi_start:] = 3e38 if kind.startswith("huge") else np.inf
    return s if n > 10 ** 6 else s[np.random.default_rng(seed).permutation(n)]


@lru_cache(maxsize=1)
def _ramp(n):
    """Sorted distinct-ish values: the infinity placements need no partition on it."""
    return np.linspace(-1.0, 1.0, n, dtype=F32)


def _with_nan(a, bits, at):
    b = a.copy()
    b[at] = np.array([bits], np.uint32).view(F32)[0]
    return b


def _pcts(n):
    rng = np.random.default_rng(1000 + n)
    return PCTS + tuple(float(x) for x in rng.uniform(0, 100, 1 if n > 10 ** 6 else 8))


def _cases(n):
    """(label, values, percent) over the whole matrix for one size; fewer variants at the multi-million sizes."""
    a = _base(n)
    big = n > 10 ** 6
    for p in _pcts(n):
        yield f"p={p!r}", a, p
    for p in ((50.0,) if big else _pcts(n)):
        for kind in (("lo_at", "hi_next", "both_at") if big else
                     ("lo_at", "hi_at", "both_at", "lo_next", "hi_next", "both_next")):
            yield f"{kind} p={p!r}", _with_infs(a, p, kind, seed=n), p
    for i, bits in enumerate(NANS[:1] if big else NANS):
        for at in ((n - 1,) if big else (0, n - 1, n // 2)):
            yield f"nan {bits:#x} at {at}", _with_nan(a, bits, at), (50.0, 99.9, 0.0)[i % 3]
    if n >= 2 ** 24 - 1:          # around 2^24 the ranks round in fp32: every percent, at and beside the selected ranks
        for p in _pcts(n):
            for kind in ("lo_at", "hi_at", "hi_next", "huge_at"):
                yield f"ramp {kind} p={p!r}", _with_infs(_ramp(n), p, kind, seed=n, is_sorted=True), p


def _same(x, y):
    """Bit-equal fp32 scalars, any NaN equal to any NaN."""
    x, y = F32(x), F32(y)
    if np.isnan(x) or np.isnan(y):
        return bool(np.isnan(x) and np.isnan(y))
    return x.view(np.uint32) == y.view(np.uint32)


@needs_numpy2
@pytest.mark.parametrize("n", SIZES)
def test_percentile_f32_is_numpys_percentile(n):
    bad = []
    with np.errstate(invalid="ignore", over="ignore"):
        for label, a, p in _cases(n):
            t = np.percentile(a, p)
            r = percentile_f32(a, p)
            assert isinstance(r, np.float32) and np.asarray(t).dtype == np.float32, (label, type(r), type(t))
            if not _same(r, t):
                bad.append((label, float(r), float(t)))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ percentile and mask on the device
def _device_mask(a, p, floor):
    from omnivggt_official_b200 import ops
    mask, thr, cnt = ops.conf_percentile_mask(torch.from_numpy(np.ascontiguousarray(a)).cuda(), p, floor=floor)
    torch.cuda.synchronize()
    return mask.cpu().numpy().astype(bool), F32(thr.item()), int(cnt.item())


def _check_mask(label, a, p, floor, bad):
    m, t, c = _device_mask(a, p, floor)
    t_ref = percentile_f32(a, p)
    with np.errstate(invalid="ignore"):
        m_ref = (a >= t_ref) & (a > F32(floor))
    if not _same(t, t_ref):
        bad.append((label, "threshold", float(t), float(t_ref)))
    elif not np.array_equal(m, m_ref):
        bad.append((label, "mask", int((m != m_ref).sum())))
    elif c != int(m_ref.sum()):
        bad.append((label, "count", c, int(m_ref.sum())))


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_conf_percentile_mask_is_numpys(n):
    bad = []
    for label, a, p in _cases(n):
        _check_mask(label, a, p, 0.1, bad)
    assert not bad, bad


def _shared_bits(n, keep, seed):
    """n values whose keys share their top `keep` bits: every radix pass down to bit `keep` splits one full bucket."""
    rng = np.random.default_rng(seed)
    low = rng.integers(0, 1 << (32 - keep), n, dtype=np.uint32)
    return ((np.uint32(0x3F9A5C3E) & np.uint32((0xFFFFFFFF << (32 - keep)) & 0xFFFFFFFF)) | low).view(F32)


@pytest.mark.gpu
def test_conf_percentile_mask_edges():
    """Equal values, all NaN, one NaN at the last index, values that share their top 8 / 16 / 24 key bits, and the floors."""
    bad = []
    rng = np.random.default_rng(7)
    cases = []
    for n in (1, 2, 3, 5, 6, 1027, VIEWS8 + 3):
        cases.append((f"equal n={n}", np.full(n, 1.25, F32)))
        cases.append((f"all nan n={n}", np.full(n, np.nan, F32)))
        cases.append((f"nan last n={n}", _with_nan((1 + rng.random(n)).astype(F32), 0x7FC00000, n - 1)))
        cases.append((f"-nan last n={n}", _with_nan((1 + rng.random(n)).astype(F32), 0xFFC00000, n - 1)))
    for keep in (8, 16, 24):
        for n in (4099, VIEWS8):
            cases.append((f"top {keep} bits n={n}", _shared_bits(n, keep, keep + n)))
            neg = -_shared_bits(n, keep, keep + n + 1)
            cases.append((f"top {keep} bits negative n={n}", neg))
    for label, a in cases:
        for p in (0.0, 12.5, 50.0, 99.9, 100.0):
            _check_mask(f"{label} p={p}", a, p, 0.1, bad)
    big = (np.exp(rng.standard_normal(VIEWS24)) * 1e-4).astype(F32)
    big[::13] = 1e-5
    for floor in (0.1, 1e-5, -1e30):
        for n, a in ((9, big[:9]), (VIEWS8, big[:VIEWS8]), (VIEWS24, big)):
            for p in (25.0, 50.0):
                _check_mask(f"floor={floor} n={n} p={p}", a, p, floor, bad)
    assert not bad, bad


# ----------------------------------------------------------------------------------------------------- point cloud centre / scale
def _sel_offset():
    """Byte offset of the scale's [6][3] selection results in the point-cloud workspace.  cloud_layout (csrc/ovg.cu) carves
    the percentile region of OVG_PERCENTILE_WORKSPACE_BYTES first and these 18 floats next, each buffer starting on a
    256-byte boundary (Arena::take)."""
    from omnivggt_official_b200 import _lib as L
    return (L.PERCENTILE_WORKSPACE_BYTES + 255) // 256 * 256


@pytest.mark.gpu
@pytest.mark.parametrize("n", (1, 2, 5, 1001, 2 ** 20 + 3, VIEWS8))
def test_point_cloud_center_and_scale(n):
    from omnivggt_official_b200 import ops
    rng = np.random.default_rng(n)
    pts = np.stack([rng.standard_normal(n) * 3 + 40,                        # an offset: the mean is not small
                    rng.standard_normal(n) * np.exp(rng.standard_normal(n)),
                    np.round(rng.standard_normal(n) * 4) / 4 - 1e4], -1).astype(F32)   # ties
    dp = torch.from_numpy(pts).cuda()
    ws = ops.point_cloud_workspace(n, dp.device)
    center = ops.point_cloud_center(dp, ws).cpu().numpy()
    # fp64 partial sums: one run per thread over n / (256 x 256) points, a 256-way tree, a 256-term sum, one division
    steps = n / 65536 + 8 + 256 + 2
    for a in range(3):
        x = pts[:, a].astype(np.float64)
        m = math.fsum(x) / n
        bound = 0.5 * float(np.spacing(abs(F32(m)))) + steps * 2.0 ** -53 * float(np.abs(x).sum()) / n
        assert abs(float(center[a]) - m) <= bound, (a, float(center[a]), m, bound)
    ld = (n + 3) // 4 * 4
    xyz = torch.full((3, ld), float("nan"), device="cuda")
    xyz[:, :n] = dp.t()
    scale = F32(ops.point_cloud_scale(xyz, n, ws).item())
    off = _sel_offset()
    sel = ws[off:off + 72].view(torch.float32).cpu().numpy().reshape(2, 3, 3)
    # the selected pairs must be order statistics of the column: if they are not, the offset no longer finds them
    cols = np.sort(pts, axis=0)
    assert all(np.isin(sel[i, a, :2], cols[:, a]).all() for i in range(2) for a in range(3)), \
        ("the scale's selection results are not at the expected workspace offset (see _sel_offset)", sel)
    q = np.array([[percentile_f32(pts[:, a], p) for a in range(3)] for p in (5.0, 95.0)], F32)
    assert all(_same(sel[i, a, 2], q[i, a]) for i in range(2) for a in range(3)), (sel[..., 2], q)
    ref = np.linalg.norm(q[1] - q[0])
    assert ref.dtype == F32 and abs(float(scale) - float(ref)) <= float(np.spacing(ref)), (scale, ref)


# --------------------------------------------------------------------------------------------------------------- pose decode
def _lib():
    from omnivggt_official_b200 import _lib as L
    return L


def _pose_inputs(K, seed):
    rng = np.random.default_rng(seed)
    pe = np.empty((K, 9), F32)
    pe[:, :3] = rng.standard_normal((K, 3)) * np.exp(rng.uniform(-3, 3, (K, 1)))
    q = rng.standard_normal((K, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q *= 10.0 ** rng.uniform(-3, 3, (K, 1))                                   # norms 1e-3 .. 1e3
    q[::2, 3] = np.abs(q[::2, 3])                                             # both signs of the real part
    q[1::2, 3] = -np.abs(q[1::2, 3])
    pe[:, 3:7] = q
    fovs = np.array([1e-6, 0.1, 1.0, 2.5, math.pi - 1e-3, 0.0], F32)
    pe[:, 7] = fovs[np.arange(K) % fovs.size]
    pe[:, 8] = fovs[(np.arange(K) + 2) % fovs.size]
    if K > 1:
        pe[K // 2, 3:7] = 0.0                                                 # zero quaternion: NaN on both sides
    return pe


def _pose_ref(pe, H, W):
    """fp64 of the kernel's formulas from the fp32 inputs, and each element's magnitude sum M (terms before cancelling)."""
    x = pe.astype(np.float64)
    t, (i, j, k, r) = x[:, :3], x[:, 3:7].T
    with np.errstate(divide="ignore", invalid="ignore"):
        s2 = 2.0 / (i * i + j * j + k * k + r * r)
        R = np.stack([1 - s2 * (j * j + k * k), s2 * (i * j - k * r), s2 * (i * k + j * r),
                      s2 * (i * j + k * r), 1 - s2 * (i * i + k * k), s2 * (j * k - i * r),
                      s2 * (i * k - j * r), s2 * (j * k + i * r), 1 - s2 * (i * i + j * j)], -1).reshape(-1, 3, 3)
        M = np.stack([1 + s2 * (j * j + k * k), s2 * (abs(i * j) + abs(k * r)), s2 * (abs(i * k) + abs(j * r)),
                      s2 * (abs(i * j) + abs(k * r)), 1 + s2 * (i * i + k * k), s2 * (abs(j * k) + abs(i * r)),
                      s2 * (abs(i * k) + abs(j * r)), s2 * (abs(j * k) + abs(i * r)), 1 + s2 * (i * i + j * j)],
                     -1).reshape(-1, 3, 3)
        fy = (H / 2.0) / np.tan(x[:, 7] / 2.0)
        fx = (W / 2.0) / np.tan(x[:, 8] / 2.0)
        Rt = np.swapaxes(R, 1, 2)
        ct = -(Rt @ t[:, :, None])[..., 0]
    return R, M, t, fx, fy, ct


def _pose_device(pe, H, W, with_intrinsic=True, with_cam2world=True):
    L = _lib()
    K = pe.shape[0]
    d = torch.from_numpy(pe).cuda()
    ext = torch.full((K, 3, 4), float("nan"), device="cuda")
    intr = torch.full((K, 3, 3), float("nan"), device="cuda")
    c2w = torch.full((K, 3, 4), float("nan"), device="cuda")
    L.check(L.lib().ovg_pose_decode(d.data_ptr(), ext.data_ptr(), intr.data_ptr() if with_intrinsic else None,
                                    c2w.data_ptr() if with_cam2world else None, K, H, W, L.stream()))
    torch.cuda.synchronize()
    return ext.cpu().numpy(), intr.cpu().numpy(), c2w.cpu().numpy()


def _within(got, ref, bound):
    """Per element: equal non-finite values (NaN to NaN, infinities by sign), else |got - ref| <= bound."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    fin = np.isfinite(ref)
    same = (np.isnan(got) & np.isnan(ref)) | (got == ref)
    ok = np.where(fin, np.abs(got - np.where(fin, ref, 0)) <= bound, same)
    return ok


@pytest.mark.gpu
@pytest.mark.parametrize("K", (1, 127, 128, 129, 4096))
@pytest.mark.parametrize("HW", ((518, 518), (294, 518), (518, 378)))
def test_pose_decode_per_element(K, HW):
    H, W = HW
    pe = _pose_inputs(K, seed=K + H)
    ext, intr, c2w = _pose_device(pe, H, W)
    R, M, t, fx, fy, ct = _pose_ref(pe, H, W)
    # R: s = i^2 + j^2 + k^2 + r^2 (4 roundings), 2 / s (1), the pair product / sum (2), the product with 2 / s (1), 1 - x
    # (1): |error| <= 9 u M (M: the terms' magnitudes), and 10 u M leaves a margin for the gamma_n second-order terms.
    assert _within(ext[:, :, :3], R, 10 * U * M).all()
    assert np.array_equal(ext[:, :, 3], pe[:, :3])                                        # t copied
    # fx = (W / 2) / tanf(fov / 2): W / 2 and fov / 2 are exact, tanf is within 4 ulp, the division rounds once
    f_ref = np.stack([fx, fy], -1)
    f_got = np.stack([intr[:, 0, 0], intr[:, 1, 1]], -1)
    assert _within(f_got, f_ref, 6 * U * np.abs(np.where(np.isfinite(f_ref), f_ref, 0))).all()
    assert (intr[pe[:, 8] == 0, 0, 0] == np.inf).all() and (intr[pe[:, 7] == 0, 1, 1] == np.inf).all()
    rest = intr.reshape(K, 9)[:, [1, 2, 3, 5, 6, 7, 8]]
    assert np.array_equal(rest, np.tile(np.array([0, W / 2, 0, H / 2, 0, 0, 1], F32), (K, 1)))
    # cam2world: R^T copied bit for bit from the extrinsic; -(R^T t) with R's error carried through plus a 3-term dot (3 u)
    assert np.array_equal(c2w[:, :, :3], np.swapaxes(ext[:, :, :3], 1, 2), equal_nan=True)
    Mt = np.swapaxes(M, 1, 2)
    ct_bound = ((10 * U * Mt + 4 * U * np.abs(np.swapaxes(R, 1, 2))) * np.abs(t)[:, None, :]).sum(-1)
    assert _within(c2w[:, :, 3], ct, ct_bound).all()
    zero = ~np.any(pe[:, 3:7], axis=1)
    assert np.isnan(ext[zero, :, :3]).all() and np.isnan(R[zero]).all()


@pytest.mark.gpu
def test_pose_decode_null_outputs():
    """intrinsic and cam2world may be NULL: the extrinsic is the same, and the other outputs are not touched."""
    pe = _pose_inputs(129, seed=3)
    ext, intr, c2w = _pose_device(pe, 294, 518)
    for wi, wc in ((False, True), (True, False), (False, False)):
        e2, i2, c2 = _pose_device(pe, 294, 518, wi, wc)
        assert np.array_equal(e2, ext, equal_nan=True)
        assert np.array_equal(i2, intr, equal_nan=True) if wi else np.isnan(i2).all()
        assert np.array_equal(c2, c2w, equal_nan=True) if wc else np.isnan(c2).all()


# ---------------------------------------------------------------------------------------------------------------- unproject
def _cameras(K, H, W, seed):
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((K, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    i, j, k, r = q.T
    R = np.stack([1 - 2 * (j * j + k * k), 2 * (i * j - k * r), 2 * (i * k + j * r),
                  2 * (i * j + k * r), 1 - 2 * (i * i + k * k), 2 * (j * k - i * r),
                  2 * (i * k - j * r), 2 * (j * k + i * r), 1 - 2 * (i * i + j * j)], -1).reshape(K, 3, 3)
    c2w = np.concatenate([R, rng.standard_normal((K, 3, 1)) * 5], -1).astype(F32)
    c2w[::3, :, 3] = 0.0                                                      # no translation: nothing hides an error
    intr = np.zeros((K, 3, 3), F32)
    intr[:, 0, 0] = rng.uniform(0.3, 3, K) * W
    intr[:, 1, 1] = rng.uniform(0.3, 3, K) * H
    intr[1::4, 0, 0] = np.inf                                                  # fov 0: the untrained model's focal lengths
    intr[1::4, 1, 1] = np.inf
    intr[:, 0, 2], intr[:, 1, 2], intr[:, 2, 2] = W / 2, H / 2, 1
    return intr, c2w


def _depths(K, H, W, seed):
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.1, 10, (K, H, W)).astype(F32).reshape(-1)
    special = np.array([0.0, 1e-40, -2.5, 1e30, np.inf, -0.0], F32)
    d[:min(d.size, special.size)] = special[:d.size]
    at = rng.integers(0, d.size, min(d.size, 4096))
    d[at] = special[rng.integers(0, special.size, at.size)]
    return d.reshape(K, H, W)


def _unproject_ref(depth, intr, c2w):
    """fp64 world points and, per coordinate, the bound 8 u (sum_j |r_ij c_j| + |t_i|) + 8 eta: the camera coordinates carry
    3 roundings ((u - cu) d, x 1 / fu and 1 / fu itself), the 3-term dot product plus t 4 more, and each of those operations
    may lose one eta to underflow."""
    K, H, W = depth.shape
    d = depth.astype(np.float64)
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    fu, fv = intr[:, 0, 0].astype(np.float64), intr[:, 1, 1].astype(np.float64)
    cu, cv = intr[:, 0, 2].astype(np.float64), intr[:, 1, 2].astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        x = (u - cu[:, None, None]) * d * (1.0 / fu)[:, None, None]
        y = (v - cv[:, None, None]) * d * (1.0 / fv)[:, None, None]
        cam = np.stack([x, y, d], -1)
        R, t = c2w[:, :, :3].astype(np.float64), c2w[:, :, 3].astype(np.float64)
        terms = cam[..., None, :] * R[:, None, None, :, :]                      # [K, H, W, 3 (i), 3 (j)]
        world = ((terms[..., 0] + terms[..., 1]) + terms[..., 2]) + t[:, None, None, :]
        bound = 8 * U * (np.abs(terms).sum(-1) + np.abs(t)[:, None, None, :]) + 8 * ETA
    return world, bound


@pytest.mark.gpu
@pytest.mark.parametrize("KHW", ((1, 1, 1), (2, 3, 5), (3, 4, 6), (2, 5, 8), (1, 518, 518), (24, 518, 518), (3, 882, 518),
                                 (65535, 1, 4)))
def test_unproject_depth_per_element(KHW):
    """(3, 4, 6): H W % 4 == 0 but W % 4 != 0 takes the scalar path, (2, 5, 8) the float4 path; (24, 518, 518) and
    (3, 882, 518) cap the grid at 8 blocks per SM over the frames, so the grid-stride loop runs."""
    L = _lib()
    K, H, W = KHW
    depth = _depths(K, H, W, seed=K * 7 + H)
    intr, c2w = _cameras(K, H, W, seed=K + W)
    dd = torch.from_numpy(depth).cuda()
    di, dc = torch.from_numpy(intr).cuda(), torch.from_numpy(c2w).cuda()
    world = torch.full((K, H, W, 3), float("nan"), device="cuda")
    L.check(L.lib().ovg_unproject_depth(dd.data_ptr(), di.data_ptr(), dc.data_ptr(), world.data_ptr(), K, H, W, L.stream()))
    torch.cuda.synchronize()
    got = world.cpu().numpy()
    ref, bound = _unproject_ref(depth, intr, c2w)
    ok = _within(got, ref, bound)
    assert ok.all(), [(tuple(i), float(got[tuple(i)]), float(ref[tuple(i)]), float(bound[tuple(i)]))
                      for i in np.argwhere(~ok)[:8]]
    finite = np.isfinite(depth) & np.isfinite(intr[:, 0, 0])[:, None, None]
    assert np.isfinite(got[finite]).all()                                   # no element left at its NaN fill
