"""The kernels that produce every depth and point map, against the fp64 references of oracle/kernel_ref.py, element by element:
the fused DPT output tail (ovg_dpt_tail: fusedtail_kernel + tail_tables_kernel), ovg_upsample_bilinear (rows and direct kernels),
ovg_im2col3x3s2, ovg_image_im2col and ovg_depth_im2col.

Exact tier: geometries whose sample positions are dyadic, small-integer maps and dyadic weights make every fp32 step exact (the
test asserts the conditions on the CPU), so outputs must equal the reference bit for bit, or within the fp32 libm error after the
exact pre-activation.  Bound tier: the shapes the model runs, within per-element bounds, each printing its margin.  Every output
sits between sentinel guards; work splits that depend on the SM count are derived from this device's."""
import pytest
import torch
import torch.nn.functional as Fn

from oracle import kernel_ref as R
from ovg_support import guarded, guards_ok, lib_module, margin, ops_module

pytestmark = pytest.mark.gpu

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
SENT = -7.0e30          # fp32 sentinel: an element the kernel should have written and did not is far outside any bound


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _kernels(fn):
    """Names of the CUDA kernels `fn` launches (torch.profiler).  The profiler now and then drops device records, all of them
    or only some (a trace with the fused tail but without the tables kernel launched just before it); it never invents one.
    `fn` is idempotent, so it is profiled three times and the names of all traces are returned."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    names = set()
    for i in range(10):       # and up to seven more times while every trace came back empty
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names |= {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
        if i >= 2 and names:
            break
    assert names, "the profiler recorded no kernel"
    return names


def _ran(names, kernel):
    return any(kernel in n for n in names)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _dyadic_bits(n_src, n_dst):
    """Fractional bits of the kernels' sample positions (None if not all are dyadic with <= 8 bits)."""
    *_, f = R.sample_positions(n_src, n_dst)
    for b in range(9):
        if torch.equal(torch.round(f * 2 ** b), f * 2 ** b):
            return b
    return None


# ----------------------------------------------------------------------------------------------- upsampling
def _upsample(src, H, W, tx, ty, dtype, fill=-3.0):
    """ovg_upsample_bilinear on the interior src [F, h, w, C] (cpu fp64 / 16-bit values), output between guards.  Returns the
    interior [F, H, W, C] and the kernels launched; asserts the border is zero and the guards are intact."""
    ops = ops_module()
    Fr, h, w, C = src.shape
    xp = Fn.pad(src.to(F64), (0, 0, 1, 1, 1, 1)).to(dtype).cuda()
    buf, flat = guarded(Fr * (H + 2) * (W + 2) * C, dtype, fill)
    txd = tx.float().cuda() if tx is not None else None
    tyd = ty.float().cuda() if ty is not None else None
    names = _kernels(lambda: ops.upsample_bilinear(xp, flat, txd, tyd, Fr, h, w, H, W, C))
    out = flat.view(Fr, H + 2, W + 2, C)
    border = out.clone()
    border[:, 1:-1, 1:-1] = 0
    assert (border == 0).all() and guards_ok(buf, fill)
    want = "upsample_rows_kernel" if R.upsample_path(w, C) == "rows" else "upsample_bilinear_kernel"
    assert _ran(names, want) and not _ran(names, "upsample_rows_kernel" if want != "upsample_rows_kernel" else
                                          "upsample_bilinear_kernel"), names
    return out[:, 1:-1, 1:-1], want


# (h, w, H, W): dyadic (w-1)/(W-1) and (h-1)/(H-1): 1/2, 1/4, 1/8, 3/8, 5/16 and 1 (h = H)
EXACT_GEOMS = [(3, 5, 5, 9), (2, 129, 3, 257), (3, 97, 5, 385), (4, 49, 4, 385), (5, 6, 9, 17), (4, 4, 4, 9), (9, 37, 17, 73)]


def _exact_inputs(Fr, h, w, H, W, C, seed, tables=True):
    """Small-integer map, tables in units of the output's lsb: the blend, the table add and the 16-bit store are exact."""
    b = _dyadic_bits(h, H) + _dyadic_bits(w, W)
    assert b <= 7
    g = _gen(seed)
    V = min(8, 2 ** (7 - b))
    src = torch.randint(-V, V + 1, (Fr, h, w, C), generator=g).to(F64)
    tx = ty = None
    if tables:
        tx = torch.randint(-64, 65, (W, C // 2), generator=g).to(F64) * 2.0 ** -b
        ty = torch.randint(-64, 65, (H, C // 2), generator=g).to(F64) * 2.0 ** -b
    return src, tx, ty, b


@pytest.mark.parametrize("tables", [False, True])
@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("C", [128, 48])
@pytest.mark.parametrize("h,w,H,W", EXACT_GEOMS)
def test_upsample_exact(h, w, H, W, C, dtype, tables):
    """Both kernels (C = 128: rows, C = 48: direct), with and without tables: bit for bit on exact geometries."""
    src, tx, ty, b = _exact_inputs(2, h, w, H, W, C, seed=h * 1000 + W, tables=tables)
    ref, _ = R.bilinear_ref(src, H, W, tx, ty, dtype)
    assert torch.equal(R.round_to(ref, dtype), ref) and torch.equal(ref.float().double(), ref)      # exact by construction
    out, path = _upsample(src, H, W, tx, ty, dtype)
    bad = (out.double().cpu() != ref).nonzero()
    assert bad.numel() == 0, f"{path}: {bad.shape[0]} mismatches, first (frame, y, x, c) {tuple(bad[0].tolist())}"


UP_BOUND = [  # (name, F, h, w, H, W, C, tables, dtype)
    ("fusion 19->37", 2, 19, 19, 37, 37, 256, False, F16),
    ("fusion 37->74", 2, 37, 37, 74, 74, 256, False, BF16),
    ("fusion 74->148", 2, 74, 74, 148, 148, 256, False, F16),
    ("fusion 148->296", 1, 148, 148, 296, 296, 256, False, BF16),
    ("fusion 16->28x18->32", 2, 16, 18, 28, 32, 256, False, BF16),
    # the first fusion of the 294-, 392- and 882-pixel-high inputs at a 518-pixel width (stride-2 level -> patch grid)
    ("fusion 11x19->21x37", 2, 11, 19, 21, 37, 256, False, F16),
    ("fusion 14x19->28x37", 2, 14, 19, 28, 37, 256, False, BF16),
    ("fusion 32x19->63x37", 2, 32, 19, 63, 37, 256, False, F16),
    ("tail 148->296 tables", 1, 148, 148, 296, 296, 128, True, F16),
    ("direct C=48", 2, 8, 12, 14, 21, 48, True, BF16),
    ("direct C=144", 2, 19, 19, 37, 37, 144, True, F16),
    ("direct w=400", 1, 4, 400, 7, 700, 64, True, BF16),
    ("direct w=400 fp16", 1, 5, 401, 9, 803, 128, False, F16),
]


@pytest.mark.parametrize("name,Fr,h,w,H,W,C,tables,dtype", UP_BOUND, ids=[u[0] for u in UP_BOUND])
def test_upsample_bound(name, Fr, h, w, H, W, C, tables, dtype):
    g = _gen(W + C)
    src = torch.randn(Fr, h, w, C, generator=g, dtype=F64).to(dtype).to(F64)
    tx = torch.randn(W, C // 2, generator=g).float() * 0.1 if tables else None
    ty = torch.randn(H, C // 2, generator=g).float() * 0.1 if tables else None
    out, path = _upsample(src, H, W, tx, ty, dtype)
    ref, bound = R.bilinear_ref(src.cuda(), H, W, tx, ty, dtype)
    r, f = R.check_rounded(out, ref, bound, dtype, f"upsample {name} ({path})", ("frame", "y", "x", "c"))
    margin(f"upsample {name} {dtype} ({path})", r)
    print(f"  equal to round(ref): {f:.5f}")


@pytest.mark.parametrize("C", [64, 48])
def test_upsample_fp16_saturates(C):
    """A blend plus table above 65504 is stored as +-65504, never inf, on both kernels."""
    h, w, H, W = 3, 4, 5, 7
    src = torch.full((1, h, w, C), 65504.0, dtype=F64)
    src[..., 1::2] = -65504.0
    tx = torch.full((W, C // 2), 64.0)
    tx[:, 1::2] = -64.0
    ty = torch.full((H, C // 2), 64.0)
    ty[:, 1::2] = -64.0
    out, path = _upsample(src, H, W, tx, ty, F16)
    out = out.float().cpu()
    assert torch.isfinite(out).all(), path
    assert (out[..., 0::2] == 65504).all() and (out[..., 1::2] == -65504).all(), path


# ----------------------------------------------------------------------------------------------- fused DPT tail
def _tail(src, tx, ty, wb, b1, w2, b2, act, H, W, dtype, names=False):
    """ovg_dpt_tail through the C entry point: guarded preds, conf and scratch.  Returns (preds, conf, gx, gy) on the device
    (gx, gy: the tables read back from the scratch; None without tables)."""
    L = lib_module()
    Fr, h, w, C = src.shape
    outc = w2.shape[0]
    xp = Fn.pad(src.to(F64), (0, 0, 1, 1, 1, 1)).to(dtype).cuda().contiguous()
    wbd = wb.to(dtype).cuda().contiguous()
    b1d, w2d, b2d = b1.float().cuda(), w2.float().cuda().contiguous(), b2.float().cuda()
    txd = tx.float().cuda().contiguous() if tx is not None else None
    tyd = ty.float().cuda().contiguous() if ty is not None else None
    pbuf, preds = guarded(Fr * H * W * (outc - 1), F32, SENT)
    cbuf, conf = guarded(Fr * H * W, F32, SENT)
    sbuf, scratch = guarded(L.lib().ovg_dpt_tail_scratch_bytes(H, W) // 4, F32, SENT)

    def run():
        L.check(L.lib().ovg_dpt_tail(xp.data_ptr(), L.ptr(txd), L.ptr(tyd), wbd.data_ptr(), b1d.data_ptr(), w2d.data_ptr(),
                                     b2d.data_ptr(), outc, act, preds.data_ptr(), conf.data_ptr(), Fr, h, w, H, W,
                                     int(dtype == F16), scratch.data_ptr(), L.stream()))
    ks = _kernels(run) if names else None
    if not names:
        run()
    torch.cuda.synchronize()
    assert guards_ok(pbuf, SENT) and guards_ok(cbuf, SENT) and guards_ok(sbuf, SENT)
    if ks is not None:
        assert _ran(ks, "fusedtail_kernel") and _ran(ks, "tail_tables_kernel") == (tx is not None), ks
    gx = gy = None
    if tx is not None:
        gx = scratch[:3 * W * 32].view(3, W, 32)
        gy = scratch[3 * W * 32:3 * (W + H) * 32].view(3, H, 32)
    else:
        assert (scratch == SENT).all()
    return preds.view(Fr, H, W, outc - 1), conf.view(Fr, H, W), gx, gy


TAIL_EXACT = [  # (h, w, H, W, outc, act, dtype, tables)
    (3, 5, 5, 9, 2, 0, BF16, True),
    (2, 129, 3, 257, 3, 1, F16, True),
    (3, 97, 5, 385, 4, 0, F16, True),
    (4, 49, 4, 385, 4, 1, BF16, True),
    (5, 6, 9, 17, 3, 0, BF16, True),
    (9, 37, 17, 73, 2, 1, F16, True),
    (2, 129, 3, 257, 4, 1, BF16, False),
    (9, 37, 17, 73, 3, 0, BF16, True),
    (3, 5, 5, 9, 4, 1, F16, False),
]


@pytest.mark.parametrize("h,w,H,W,outc,act,dtype,tables", TAIL_EXACT)
def test_dpt_tail_exact(h, w, H, W, outc, act, dtype, tables, sms):
    """Exact pre-activation: the tables equal tail_tables_ref bit for bit, and preds / conf equal exp / sign expm1 / 1 + exp of
    the fp64 pre-activation within the fp32 libm error.  F = 3; several strips and a one-pixel last strip (W = 128 k + 1);
    seg_rows < 8 (H < 8); h = H (sy = 1); 1/8 steps (the n > 2 emit loop)."""
    Fr = 3
    sch = R.tail_schedule(Fr, H, W, sms)
    if W > 128:
        assert sch["n_strips"] >= 3 and sch["last_strip_px"] == 1, sch
    if H < 8:
        assert sch["seg_rows"] < 8, sch
    assert R.tail_supported(h, w, H, W) and lib_module().lib().ovg_dpt_tail_supported(h, w, H, W, 128) == 1
    src, _, _, b = _exact_inputs(Fr, h, w, H, W, 128, seed=h * 100 + W)
    g = _gen(W)
    qt = 4
    tx = torch.randint(-8, 9, (W, 64), generator=g).to(F64) / 2 ** qt if tables else None
    ty = torch.randint(-8, 9, (H, 64), generator=g).to(F64) / 2 ** qt if tables else None
    wb = torch.randint(-2, 3, (32, 9 * 128), generator=g).to(F64)
    b1 = torch.randint(-16, 17, (32,), generator=g).to(F64) / 16
    w2 = torch.randint(-3, 4, (outc, 32), generator=g).to(F64) / 256
    b2 = torch.randint(-64, 65, (outc,), generator=g).to(F64) / 256
    # exactness conditions: the resized operand fits the 16-bit type; conv, table and 1x1 partial sums stay below 2^24 lsb
    up, _, _ = R._blend(src, H, W)
    assert torch.equal(R.round_to(up, dtype), up)
    qh = max(b, qt)
    wk = wb.reshape(32, 3, 3, 128)
    emb = R.embedding_map(tx, ty, H, W, 128)[None]
    hx = R.conv3x3(up + emb, wk) + b1
    habs = R.conv3x3(up.abs() + emb.abs(), wk.abs()) + b1.abs()
    assert float(habs.max()) * 2 ** qh < 2 ** 24
    assert torch.equal(torch.round(hx * 2 ** qh), hx * 2 ** qh)
    assert float((hx.clamp(min=0) @ w2.abs().t() + b2.abs()).max()) * 2 ** (qh + 8) < 2 ** 24
    preds, conf, gx, gy = _tail(src, tx, ty, wb, b1, w2, b2, act, H, W, dtype, names=True)
    rp, rc, bp, bc = R.head_post(hx, torch.zeros_like(hx), w2, b2, act, epi_c=0.0)
    if tables:
        rgx, rgy = R.tail_tables_ref(tx, ty, wb, H, W)
        assert torch.equal(gx.double().cpu(), rgx) and torch.equal(gy.double().cpu(), rgy)
    r1 = R.check_bound(preds, rp, bp, "tail preds (exact tier)", ("frame", "y", "x", "c"))
    r2 = R.check_bound(conf, rc, bc, "tail conf (exact tier)", ("frame", "y", "x"))
    margin(f"dpt tail exact {h}x{w}->{H}x{W} outc={outc} act={act} {dtype} (libm ulps / 2)", max(r1, r2))


def _span(w, W):
    import numpy as np
    return int((np.float32(w - 1) / np.float32(W - 1)) * np.float32(129.0)) + 3


def _span80_W(w):
    """The smallest W (largest sx) that ovg_dpt_tail_supported accepts for w: its strips span exactly 80 source pixels."""
    for W in range(w + 1, 4 * w):
        if R.tail_supported(2, w, 2, W):
            return W
    raise AssertionError(w)


TAIL_BOUND = [  # (name, F, h, w, H, W, outc, act, dtype, tables)
    ("518 F=1", 1, 296, 296, 518, 518, 2, 0, BF16, True),
    ("518 F=3", 3, 296, 296, 518, 518, 4, 1, F16, True),
    ("392x518", 2, 224, 296, 392, 518, 4, 1, BF16, True),
    ("294x518", 2, 168, 296, 294, 518, 3, 0, F16, True),
    ("882x518", 1, 504, 296, 882, 518, 4, 1, F16, True),
    ("span 80", 2, 40, 296, 70, "span80", 3, 0, F16, True),
    ("span 80 bf16", 1, 40, 200, 70, "span80", 4, 1, BF16, True),
    ("W=256", 2, 20, 148, 33, 256, 4, 1, BF16, True),
    ("W=384", 2, 20, 224, 33, 384, 2, 0, F16, True),
    ("W=641", 1, 30, 370, 52, 641, 4, 1, F16, True),
    ("W=383", 2, 30, 220, 52, 383, 3, 0, BF16, True),
    ("no tables", 2, 148, 148, 296, 296, 4, 1, BF16, False),
]


@pytest.mark.parametrize("name,Fr,h,w,H,W,outc,act,dtype,tables", TAIL_BOUND, ids=[t[0] for t in TAIL_BOUND])
def test_dpt_tail_bound(name, Fr, h, w, H, W, outc, act, dtype, tables, sms):
    if W == "span80":
        W = _span80_W(w)
        assert _span(w, W) == 80 and _span(w, W - 1) > 80
        assert lib_module().lib().ovg_dpt_tail_supported(h, w, H, W - 1, 128) == 0
    assert lib_module().lib().ovg_dpt_tail_supported(h, w, H, W, 128) == 1
    sch = R.tail_schedule(Fr, H, W, sms)
    if W in (256, 384):
        assert W - 128 * (sch["n_strips"] - 1) + 1 == 129              # zrow: the last row of the A stage
    g = torch.Generator(device="cuda").manual_seed(W + Fr)
    src = torch.randn(Fr, h, w, 128, generator=g, device="cuda", dtype=F64).to(dtype).to(F64)
    wb = (torch.randn(32, 9 * 128, generator=g, device="cuda", dtype=F64) * (9 * 128) ** -0.5).to(dtype).to(F64)
    b1 = torch.randn(32, generator=g, device="cuda").double() * 0.1
    w2 = torch.randn(outc, 32, generator=g, device="cuda").double() * 32 ** -0.5
    b2 = torch.randn(outc, generator=g, device="cuda").double() * 0.1
    tx = torch.randn(W, 64, generator=g, device="cuda") * 0.1 if tables else None
    ty = torch.randn(H, 64, generator=g, device="cuda") * 0.1 if tables else None
    b1, w2, b2 = b1.float().double(), w2.float().double(), b2.float().double()
    preds, conf, _, _ = _tail(src, tx, ty, wb, b1, w2, b2, act, H, W, dtype, names=True)
    rp, rc, bp, bc = R.dpt_tail_ref(src, tx, ty, wb, b1, w2, b2, act, H, W, dtype)
    r1 = R.check_bound(preds, rp, bp, f"tail preds {name}", ("frame", "y", "x", "c"))
    r2 = R.check_bound(conf, rc, bc, f"tail conf {name}", ("frame", "y", "x"))
    print(f"tail {name}: F={Fr} {h}x{w}->{H}x{W} schedule {sch}")
    margin(f"dpt tail {name} {dtype}", max(r1, r2))
    if Fr == 3:   # no atomics: a second run is bit-identical
        p2, c2, _, _ = _tail(src, tx, ty, wb, b1, w2, b2, act, H, W, dtype)
        assert torch.equal(p2, preds) and torch.equal(c2, conf)


# ----------------------------------------------------------------------------------------------- im2col copies
@pytest.mark.parametrize("C", [8, 256, 1024, 2048])
def test_im2col3x3s2_exact(C):
    """dst = F.unfold(pad 1, stride 2) of the NHWC input, rows (f, oy, ox) x columns (tap, c), bit for bit, between guards."""
    ops = ops_module()
    Fr = 2
    sizes = (1, 2, 3, 19, 37, 38)
    for h in sizes:
        for w in sizes:
            src = torch.randn(Fr, h, w, C, device="cuda").to(BF16)
            oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            buf, flat = guarded(Fr * oh * ow * 9 * C, BF16, -3.0)
            ops.im2col3x3s2(src, flat, Fr, h, w, C)
            u = Fn.unfold(src.float().permute(0, 3, 1, 2), 3, padding=1, stride=2)           # [F, C*9, oh*ow]
            exp = u.view(Fr, C, 9, oh * ow).permute(0, 3, 2, 1).reshape(Fr * oh * ow, 9 * C).to(BF16)
            torch.cuda.synchronize()
            got = flat.view(Fr * oh * ow, 9 * C)
            bad = (got != exp).nonzero()
            assert bad.numel() == 0, f"h={h} w={w} C={C}: first mismatch (row, col) {tuple(bad[0].tolist())}"
            assert guards_ok(buf, -3.0), (h, w, C)


# ldc 592: the DINOv2 patchifier's row stride (3 x 14^2 = 588 rounded up to a multiple of 8), at the 392- and 882-pixel-high
# inputs of a 518-pixel width
@pytest.mark.parametrize("patch,H,W,ldc", [(14, 28, 42, 608), (16, 32, 48, 784), (8, 16, 40, 200), (14, 42, 14, 592),
                                           (14, 392, 518, 592), (14, 882, 518, 592)])
def test_image_im2col_exact(patch, H, W, ldc):
    """ovg_image_im2col bit for bit against the fp32 restatement: the patch-14 template and the runtime-patch kernel, H != W,
    padding columns (ldc > 3 patch^2) pre-filled with a sentinel must come back zero."""
    L = lib_module()
    import ctypes
    K = 3
    g = torch.Generator(device="cuda").manual_seed(patch + H)
    images = torch.rand(K, 3, H, W, generator=g, device="cuda")
    mean3, std3 = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    rows = K * (H // patch) * (W // patch)
    buf, flat = guarded(rows * ldc, BF16, -3.0)
    m = (ctypes.c_float * 3)(*mean3)
    s = (ctypes.c_float * 3)(*std3)
    names = _kernels(lambda: L.check(L.lib().ovg_image_im2col(images.data_ptr(), ctypes.cast(m, ctypes.c_void_p),
                                                              ctypes.cast(s, ctypes.c_void_p), flat.data_ptr(), ldc, K, H, W,
                                                              patch, L.stream())))
    assert _ran(names, "image_im2col_kernel<14>" if patch == 14 else "image_im2col_kernel<0>"), names
    exp = R.image_cols_ref(images.cpu(), mean3, std3, patch, ldc)
    got = flat.view(rows, ldc).cpu()
    bad = (got != exp).nonzero()
    assert bad.numel() == 0, f"first mismatch (row, col) {tuple(bad[0].tolist())}: {got[tuple(bad[0])]} vs {exp[tuple(bad[0])]}"
    assert guards_ok(buf, -3.0)


def _depth_call(depth, mask, idx_stats, idx_cols, B, S, H, W, patch, ldc, fill=-3.0):
    """ovg_depth_im2col with separate view lists; returns (scale fp32 [B], cols [rows, 2 patch^2]) after checking the guards
    and the untouched columns [2 patch^2, ldc)."""
    L = lib_module()
    pp = patch * patch
    i_s = torch.tensor(idx_stats, dtype=torch.int32, device="cuda")
    i_c = torch.tensor(idx_cols, dtype=torch.int32, device="cuda")
    scratch = torch.zeros(L.DEPTH_SCRATCH_DOUBLES(B), device="cuda", dtype=F64)
    rows = B * len(idx_cols) * (H // patch) * (W // patch)
    buf, flat = guarded(rows * ldc, BF16, fill)
    names = _kernels(lambda: L.check(L.lib().ovg_depth_im2col(depth.data_ptr(), mask.data_ptr(), i_s.data_ptr(), len(idx_stats),
                                                              i_c.data_ptr(), len(idx_cols), scratch.data_ptr(), flat.data_ptr(),
                                                              ldc, B, S, H, W, patch, L.stream())))
    assert _ran(names, "depth_im2col_kernel<14>" if patch == 14 else "depth_im2col_kernel<0>"), names
    cols = flat.view(rows, ldc)
    assert guards_ok(buf, fill) and (cols[:, 2 * pp:] == fill).all()
    scale = scratch.view(F32)[2 * B * 1024 * 2:2 * B * 1024 * 2 + B].cpu()
    return scale, cols[:, :2 * pp].cpu()


def _straddling(patch):
    """(B, S, H, W, idx_stats, idx_cols): H W / 2 pairs per view, Sd H W / 2 not a multiple of DEPTH_NCHUNK = 1024 and a chunk
    span that does not divide a view, so chunks straddle views."""
    for hp in range(1, 8):
        for wp in range(1, 8):
            for sd in (7, 5, 6, 3):
                H, W = hp * patch, wp * patch
                per2, total2 = H * W // 2, H * W // 2 * sd
                span = -(-total2 // 1024)
                if hp != wp and total2 % 1024 and per2 % span:
                    stats = [0, 2, 3, 4, 5, 6, 7][:sd]
                    return 2, 8, H, W, stats, [6, 2, 3]
    raise AssertionError(patch)


@pytest.mark.parametrize("patch", [14, 16])
def test_depth_im2col_exact(patch):
    """Dyadic depths: every fp32 partial sum is exact, so the scale and the rows equal the restatement bit for bit.  The mean is
    over idx_stats, the rows over idx_cols (as when views are sharded); scene 1 has no valid pixel and must give zeros."""
    B, S, H, W, idx_stats, idx_cols = _straddling(patch)
    g = torch.Generator().manual_seed(patch)
    depth = torch.randint(128, 2049, (B, S, H, W), generator=g).float() / 256
    mask = (torch.rand(B, S, H, W, generator=g) > 0.3).float()
    mask[1] = 0
    ldc = 2 * patch * patch + 8
    scale, cols = _depth_call(depth.cuda(), mask.cuda(), idx_stats, idx_cols, B, S, H, W, patch, ldc)
    sref = R.depth_scale_ref(depth, mask, idx_stats)
    assert sref[1] == 0 and sref[0] > 0
    assert torch.equal(scale, sref), (scale, sref)
    exp = R.depth_cols_ref(depth, mask, sref, idx_cols, patch)
    bad = (cols != exp).nonzero()
    assert bad.numel() == 0, f"first mismatch (row, col) {tuple(bad[0].tolist())}"
    n1 = len(idx_cols) * (H // patch) * (W // patch)
    assert (cols[n1:] == 0).all()


DEPTH_BOUND = [  # (name, S, H, W, idx_stats, idx_cols)
    ("518x518", 8, 518, 518, list(range(8)), [1, 4, 7]),
    ("294x518", 5, 294, 518, [1, 3], [1, 3]),
]


def test_depth_im2col_bound():
    """Random depths at 518^2 (8 views) and 294 x 518 (2 of 5 views): the scale within the error of fp32 partial sums of <= 64
    values, the rows within one bf16 ulp plus that error, and >= 99 % of them equal to the fp64 value rounded once.  In both, the
    H W / 2 pairs of a view do not split evenly into the 1 024 chunks of the masked mean, so chunks straddle views."""
    B, patch = 1, 14
    for name, S, H, W, idx_stats, idx_cols in DEPTH_BOUND:
        per2 = H * W // 2
        assert per2 % -(-per2 * len(idx_stats) // 1024) != 0, name
        g = torch.Generator(device="cuda").manual_seed(5)
        depth = 0.5 + 10 * torch.rand(B, S, H, W, generator=g, device="cuda")
        mask = (torch.rand(B, S, H, W, generator=g, device="cuda") > 0.2).float()
        scale, cols = _depth_call(depth, mask, idx_stats, idx_cols, B, S, H, W, patch, 2 * patch * patch)
        d = depth.double()[:, idx_stats]
        valid = mask[:, idx_stats] > 0
        s64 = d[valid].sum()
        mean = s64 / valid.sum()
        sref = float(1.0 / (mean + 1e-8))
        rel_scale = (63 * float(d[valid].abs().sum() / s64.abs()) + 4) * R.EPS32
        r_s = abs(float(scale[0]) - sref) / (rel_scale * sref)
        assert r_s <= 1.0, (name, r_s)
        dc = depth.double()[:, idx_cols]
        ref = torch.cat([(dc * sref * mask[:, idx_cols]).reshape(-1, H // patch, patch, W // patch, patch)
                         .permute(0, 1, 3, 2, 4).reshape(-1, patch * patch),
                         mask[:, idx_cols].double().reshape(-1, H // patch, patch, W // patch, patch)
                         .permute(0, 1, 3, 2, 4).reshape(-1, patch * patch)], 1).cpu()
        bound = R.ulp(ref, BF16) + (rel_scale + 2 * R.EPS32) * ref.abs()
        r, f = R.check_rounded(cols, ref, bound, BF16, f"depth im2col rows {name}", ("row", "col"))
        margin(f"depth_im2col scale {name}", r_s)
        margin(f"depth_im2col rows {name}", r)
        print(f"  equal to round(ref): {f:.5f}")
