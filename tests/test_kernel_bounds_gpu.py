"""The GEMM, attention, LayerNorm and camera-head kernels against the fp64 references of oracle/kernel_ref.py, element by element.

Where an input can be built so that the kernel's result is exact (small integers in the GEMM; one-hot and uniform attention rows)
the test asserts bit equality.  Elsewhere every element must lie within its bound, and 16-bit outputs must equal the fp64 reference
rounded once in at least 99 % of the elements.  Each test prints its worst error as a fraction of the bound ("margin").  Shapes that
depend on the tile scheduler are derived from this device's SM count."""
import math

import pytest
import torch

from oracle import kernel_ref as R
from ovg_support import guarded, guards_ok, lib_module, margin, ops_module, randn

pytestmark = pytest.mark.gpu

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _act(x, act):
    return x.clamp(min=0) if act == "relu" else x


ACT = {"none": 0, "relu": 2}
TIES = {BF16: [257.0, 259.0, -257.0, 514.0, 1028.0, 261.0, -259.0, 263.0],
        F16: [2049.0, 2051.0, -2049.0, 4098.0, 7e4, -7e4, 65519.0, 2053.0]}    # fp16: ties, saturation, largest finite


def _int_bias(b, n, dtype):
    """Integer bias that puts row 0 (a = e_0) on the tie values: out[0, n] = b[n, 0] + bias[n]."""
    return torch.tensor([TIES[dtype][i % 8] for i in range(n)], dtype=F64) - b[:, 0]


# ----------------------------------------------------------------------------------------------- GEMM, bit exact
IDENT = [(1, 32, 8, 0), (63, 32, 56, 0), (64, 96, 72, 64), (65, 160, 392, 128), (127, 32, 4096, 0), (129, 96, 392, 64),
         (300, 160, 72, 128), (129, 256, 4096, 0)]


@pytest.mark.parametrize("act", ["none", "relu"])
@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("M,N,K,bn", IDENT)
def test_gemm_exact_ident(M, N, K, bn, dtype, act):
    """EPI_BF16, identity rows: strided A (lda > a_cols, the extra columns hold 99s), strided output (ldo > N, sentinels between
    the rows), guards around the output, row 0 on round-to-nearest-even ties (and fp16 saturation)."""
    ops = ops_module()
    a, b = R.int_operands(M, N, K, seed=M * 7 + K, extra_cols=24)
    a[:, K:] = 99.0
    a[0, :K] = 0.0
    a[0, 0] = 1.0
    bias = _int_bias(b, N, dtype)
    ldo, fill = N + 32, -3.0
    buf, flat = guarded(M * ldo, dtype, fill)
    ops.gemm(a.to(dtype).cuda()[:, :K], b.to(dtype).cuda(), epi=ops.L.EPI_BF16, bias=bias.float().cuda(), act=ACT[act],
             out=flat, ldo=ldo, block_n=bn)
    acc, _ = R.gemm_acc(a[:, :K], b)
    exp = R.round_to(_act(acc + bias[None], act), dtype)
    out = flat.view(M, ldo)
    torch.cuda.synchronize()
    assert bool(R.is_tie(acc[0] + bias, dtype).any())
    got = out[:, :N].double().cpu()
    bad = (got != exp).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} mismatches, first at (row, col) {tuple(bad[0].tolist())}: " \
                             f"{got[tuple(bad[0])]:.1f} vs {exp[tuple(bad[0])]:.1f}"
    assert (out[:, N:] == fill).all() and guards_ok(buf, fill)


@pytest.mark.parametrize("waves", ["sms-1", "sms", "sms+1", "2sms+1"])
def test_gemm_exact_scheduler_edges(waves, sms):
    """Tile counts at the edges of the persistent scheduler: SMs - 1, SMs, SMs + 1 and 2 SMs + 1 tiles of 128 x 128."""
    ops = ops_module()
    tiles = {"sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}[waves]
    M, N, K = 128 * (tiles - 1) + 1 if waves.endswith("+1") else 128 * tiles, 128, 64
    a, b = R.int_operands(M, N, K, seed=tiles)
    bias = torch.randint(-300, 300, (N,)).double()
    buf, flat = guarded(M * N, BF16, -3.0)
    ops.gemm(a.to(BF16).cuda(), b.to(BF16).cuda(), epi=ops.L.EPI_BF16, bias=bias.float().cuda(), out=flat, ldo=N, block_n=128)
    acc = (a.cuda() @ b.cuda().t())
    torch.cuda.synchronize()
    assert torch.equal(flat.view(M, N).double(), R.round_to(acc + bias.cuda()[None], BF16)) and guards_ok(buf, -3.0)


@pytest.mark.parametrize("act", ["none", "relu"])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_gemm_exact_dense2pad_table(dtype, act):
    """RM_DENSE2PAD with the additive table: rows (frame, y, x) land inside the zero-bordered map; the border stays untouched."""
    ops = ops_module()
    F, gh, gw, K, N = 3, 5, 7, 72, 96
    M = F * gh * gw
    a, b = R.int_operands(M, N, K, seed=11)
    bias = torch.randint(-200, 200, (N,)).double()
    table = torch.randint(-500, 500, (gh * gw, N)).double()
    fill = -3.0
    buf, flat = guarded(F * (gh + 2) * (gw + 2) * N, dtype, fill)
    ops.gemm(a.to(dtype).cuda(), b.to(dtype).cuda(), epi=ops.L.EPI_BF16, bias=bias.float().cuda(), act=ACT[act],
             table=table.float().cuda(), table_rows=gh * gw, out=flat, ldo=N, rowmap=ops.L.ROWS_DENSE2PAD, gh=gh, gw=gw, block_n=64)
    acc, _ = R.gemm_acc(a, b)
    exp = R.round_to(_act(acc + bias[None] + table.repeat(F, 1), act), dtype).reshape(F, gh, gw, N)
    out = flat.view(F, gh + 2, gw + 2, N)
    torch.cuda.synchronize()
    assert torch.equal(out[:, 1:-1, 1:-1].double().cpu(), exp)
    border = out.clone()
    border[:, 1:-1, 1:-1] = fill
    assert (border == fill).all() and guards_ok(buf, fill)


@pytest.mark.parametrize("act", ["none", "relu"])
@pytest.mark.parametrize("dtype", [BF16, F16])
def test_gemm_exact_pad_taps_skips(dtype, act):
    """RM_PAD, 9 row-shifted taps over a zero-bordered grid whose border rows hold non-zero values: the taps of the first and last
    rows read past both ends of a_rows (zero fill), border outputs are written as zeros, interior = taps + bias + two skips."""
    ops = ops_module()
    F, gh, gw, Cin, N = 3, 6, 9, 64, 160
    rows = F * (gh + 2) * (gw + 2)
    taps = [(ky - 1) * (gw + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    g = torch.Generator().manual_seed(12)
    a = torch.randint(-8, 9, (rows, Cin), generator=g).double()
    b = torch.randint(-8, 9, (N, 9 * Cin), generator=g).double()
    s1, s2 = (torch.randint(-64, 65, (rows, N), generator=g).double() for _ in range(2))
    bias = torch.randint(-200, 200, (N,), generator=g).double()
    fill = -3.0
    buf, flat = guarded(rows * N, dtype, fill)
    ops.gemm(a.to(dtype).cuda(), b.to(dtype).cuda(), taps=taps, epi=ops.L.EPI_BF16, bias=bias.float().cuda(), act=ACT[act],
             out=flat, ldo=N, skip1=s1.to(dtype).cuda(), skip2=s2.to(dtype).cuda(), rowmap=ops.L.ROWS_PAD, gh=gh, gw=gw, block_n=128)
    acc, _ = R.gemm_acc(a, b, taps)
    exp = R.round_to(_act(acc + bias[None] + s1 + s2, act), dtype).reshape(F, gh + 2, gw + 2, N)
    exp[:, 0], exp[:, -1], exp[:, :, 0], exp[:, :, -1] = 0.0, 0.0, 0.0, 0.0
    torch.cuda.synchronize()
    assert torch.equal(flat.view(F, gh + 2, gw + 2, N).double().cpu(), exp) and guards_ok(buf, fill)


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_gemm_exact_pixel_shuffle(dtype):
    """RM_PIXSHUF: column (ky, kx, c) of row (frame, y, x) lands at pixel (y ps + ky, x ps + kx) of the bordered output, bias and
    skip indexed by the output channel; the border stays untouched."""
    ops = ops_module()
    F, gh, gw, ps, cout, K = 2, 3, 4, 2, 32, 64
    M, N = F * gh * gw, ps * ps * cout
    a, b = R.int_operands(M, N, K, seed=13)
    bias = torch.randint(-200, 200, (cout,)).double()
    oh, ow = gh * ps + 2, gw * ps + 2
    skip = torch.randint(-64, 65, (F, oh, ow, cout)).double()
    fill = -3.0
    buf, flat = guarded(F * oh * ow * cout, dtype, fill)
    ops.gemm(a.to(dtype).cuda(), b.to(dtype).cuda(), epi=ops.L.EPI_BF16, bias=bias.float().cuda(), out=flat, ldo=cout,
             skip1=skip.to(dtype).cuda(), rowmap=ops.L.ROWS_PIXSHUF, gh=gh, gw=gw, ps=ps, cout=cout)
    acc, _ = R.gemm_acc(a, b)
    shuf = acc.reshape(F, gh, gw, ps, ps, cout).permute(0, 1, 3, 2, 4, 5).reshape(F, gh * ps, gw * ps, cout)
    exp = R.round_to(shuf + bias + skip[:, 1:-1, 1:-1], dtype)
    out = flat.view(F, oh, ow, cout)
    torch.cuda.synchronize()
    assert torch.equal(out[:, 1:-1, 1:-1].double().cpu(), exp)
    border = out.clone()
    border[:, 1:-1, 1:-1] = fill
    assert (border == fill).all() and guards_ok(buf, fill)


@pytest.mark.parametrize("M,N,K,bn", [(300, 96, 392, 64), (129, 160, 4096, 128), (65, 32, 8, 0)])
@pytest.mark.parametrize("scatter", [False, True])
def test_gemm_exact_resid(M, N, K, bn, scatter):
    """EPI_RESID: x[row] += gamma (acc + bias) in fp32, exact with integer x, acc, bias and power-of-two gamma; with row_index
    the rows are scattered through a permutation."""
    ops = ops_module()
    a, b = R.int_operands(M, N, K, seed=M + K)
    g = torch.Generator().manual_seed(N)
    bias = torch.randint(-200, 200, (N,), generator=g).double()
    gamma = torch.tensor([0.5, 2.0, -0.25, 1.0])[torch.randint(0, 4, (N,), generator=g)].double()
    x0 = torch.randint(-1000, 1000, (M, N), generator=g).double()
    perm = torch.randperm(M, generator=g)
    x = x0.float().cuda()
    ops.linear_resid(a.to(BF16).cuda(), b.to(BF16).cuda(), bias.float().cuda(), gamma.float().cuda(), x,
                     row_index=perm.int().cuda() if scatter else None, block_n=bn)
    acc, _ = R.gemm_acc(a, b)
    exp = x0.clone()
    if scatter:
        exp[perm] += gamma * (acc + bias)
    else:
        exp += gamma * (acc + bias)
    torch.cuda.synchronize()
    assert torch.equal(x.double().cpu(), exp)


@pytest.mark.parametrize("nb,ntok,C,bn", [(3, 77, 128, 0), (2, 300, 256, 64), (1, 129, 64, 0)])
def test_gemm_exact_qkv_plain(nb, ntok, C, bn):
    """EPI_QKV with qk_norm = rope = 0 (the DINOv2 blocks): bias, q times a power-of-two qscale, head-major [nb, heads, ntok, 64]
    outputs with guards."""
    ops = ops_module()
    M, heads = nb * ntok, C // 64
    a, b = R.int_operands(M, 3 * C, C, seed=ntok)
    bias = torch.randint(-200, 200, (3 * C,)).double()
    bufs = [guarded(M * C, BF16, -3.0) for _ in range(3)]
    q, k, v = (f.view(nb, heads, ntok, 64) for _, f in bufs)
    ops.gemm(a.to(BF16).cuda(), b.to(BF16).cuda(), epi=ops.L.EPI_QKV, bias=bias.float().cuda(), q_out=q, k_out=k, v_out=v, C=C,
             ntok=ntok, T=ntok, nspecial=0, wp=1, maxpos=0, qk_norm=0, rope=0, qscale=0.125, block_n=bn)
    acc, _ = R.gemm_acc(a, b)
    t = (acc + bias[None]).reshape(nb, ntok, 3, heads, 64).permute(2, 0, 3, 1, 4)
    torch.cuda.synchronize()
    assert torch.equal(q.double().cpu(), R.round_to(t[0] * 0.125, BF16))
    assert torch.equal(k.double().cpu(), R.round_to(t[1], BF16)) and torch.equal(v.double().cpu(), R.round_to(t[2], BF16))
    assert all(guards_ok(buf, -3.0) for buf, _ in bufs)


# ----------------------------------------------------------------------------------------------- GEMM, realistic inputs
def test_gemm_accumulation_constant():
    """The raw fp32 accumulator (EPI_RESID with gamma 1, bias 0 into zeros) against the exact dot products: the largest
    |acc - exact| / (sqrt(K) 2^-24 sum|a||b|) must stay at least 4x below ACC_C."""
    ops = ops_module()
    worst = 0.0
    for M, N, K in [(300, 256, 64), (1000, 384, 192), (515, 1024, 1024), (515, 1024, 4096), (2748, 1024, 1024)]:
        a = randn(M, K, seed=1, dtype=BF16)
        w = randn(N, K, scale=K ** -0.5, seed=2, dtype=BF16)
        x = torch.zeros(M, N, device="cuda")
        ops.linear_resid(a, w, torch.zeros(N, device="cuda"), torch.ones(N, device="cuda"), x)
        acc, absacc = R.gemm_acc(a, w)
        r = float(((x.double() - acc).abs() / (math.sqrt(K) * R.EPS32 * absacc)).max())
        print(f"accumulation constant, M={M} N={N} K={K}: {r:.4f}")
        worst = max(worst, r)
    margin("accumulation constant / ACC_C", worst / R.ACC_C)
    assert worst <= R.ACC_C / 4, worst


@pytest.mark.parametrize("M,N,K,bn,dtype", [(300, 256, 128, 0, BF16), (1000, 384, 192, 128, BF16), (515, 1024, 4096, 128, BF16),
                                            (77, 96, 392, 64, BF16), (2748, 3072, 1024, 512, BF16), (5000, 1024, 128, 512, BF16),
                                            (300, 256, 128, 0, F16), (2748, 1024, 1024, 512, F16)])
def test_gemm_gelu_per_element(M, N, K, bn, dtype):
    ops = ops_module()
    a = randn(M, K, seed=1, dtype=dtype)
    w = randn(N, K, scale=K ** -0.5, seed=2, dtype=dtype)
    bias = randn(N, seed=3)
    out = torch.empty(M, N, device="cuda", dtype=dtype)
    ops.gemm(a, w, epi=ops.L.EPI_BF16, bias=bias, act=ops.L.ACT_GELU, out=out, ldo=N, block_n=bn)
    ref, bound = R.linear_ref(a, w, bias, act="gelu", out_dtype=dtype)
    torch.cuda.synchronize()
    # The erf approximation of the GELU epilogue (|error| <= 1.5e-7, times |x| / 2) is within the bound, but for x < -1 it is a
    # sizable part of fp16's ulp of the small output: an fp32 emulation of it alone matches round(ref) in 99.6 % of fp16 outputs of
    # N(0, 1.3^2) inputs and 98.3 % of those below -1.  Truncating stores match about half.
    min_match = 0.97 if dtype == F16 else 0.99
    r, f = R.check_rounded(out, ref, bound, dtype, f"GEMM+GELU {M}x{N}x{K}", ("row", "col"), min_match)
    margin(f"GEMM+GELU {M}x{N}x{K} {dtype}", r)
    print(f"  equal to round(ref): {f:.5f}")


def _positions(M, T, nspecial, wp):
    t = torch.arange(M, device="cuda") % T
    pp = (t - nspecial).clamp(min=0)
    pos = torch.stack([pp // wp + 1, pp % wp + 1], -1)
    return torch.where((t >= nspecial)[:, None], pos, torch.zeros_like(pos))


def _rope_recipe(maxpos):
    """The reference's RoPE frequency tables (layers/rope.py:103-114: fp32 angles position x 100^-(2i/32), then cos and sin),
    computed on the CPU; the halves the reference concatenates are equal, so one half [maxpos, 16] is kept."""
    exponents = torch.arange(0, 32, 2).float() / 32
    inv_freq = 1.0 / (100.0 ** exponents)
    angles = torch.einsum("i,j->ij", torch.arange(maxpos, dtype=inv_freq.dtype), inv_freq)
    return angles, angles.cos(), angles.sin()


# (37, 37) and (29, 30): square and near-square 518-pixel grids; 28 x 37, 21 x 37 and 63 x 37: the 392-, 294- and 882-pixel-high
# inputs of a 518-pixel width, the last one reading row 63, the last of the 64 table rows the engine's RoPE holds.
@pytest.mark.parametrize("C,frames,hp,wp,bn", [(128, 3, 4, 4, 0), (1024, 2, 37, 37, 0), (1024, 2, 29, 30, 512), (256, 4, 3, 5, 0),
                                               (1024, 2, 28, 37, 0), (1024, 2, 21, 37, 0), (1024, 1, 63, 37, 0)])
def test_gemm_qkv_norm_rope_per_element(C, frames, hp, wp, bn):
    """EPI_QKV with LayerNorm(64) on q / k and 2-D RoPE, frame-wise sequences.  The device's RoPE tables, which the fp64
    reference takes as given, are first checked against the reference's recipe on the CPU: within 4 fp32 ulps of the angle (the
    device's pow, reciprocal and product may each round differently) plus 4 of the value (cosf / sinf)."""
    ops = ops_module()
    heads, T = C // 64, hp * wp + 5
    M = frames * T
    a = randn(M, C, seed=1, dtype=BF16)
    w = randn(3 * C, C, scale=C ** -0.5, seed=2, dtype=BF16)
    bias = randn(3 * C, scale=0.1, seed=3)
    ln = [1 + 0.1 * randn(64, seed=4), 0.1 * randn(64, seed=5), 1 + 0.1 * randn(64, seed=6), 0.1 * randn(64, seed=7)]
    maxpos = max(hp, wp) + 1
    assert maxpos <= 64
    cos, sin = ops.rope_tables(maxpos, "cuda")
    angles, rcos, rsin = _rope_recipe(maxpos)
    assert cos.shape == sin.shape == (maxpos, 16) and cos.dtype == sin.dtype == F32
    for name, got, ref in (("cos", cos, rcos), ("sin", sin, rsin)):
        bound = 4 * R.ulp(angles, F32) + 4 * R.ulp(ref, F32)
        r = R.check_bound(got, ref.double(), bound, f"RoPE {name} table, {maxpos} positions", ("position", "frequency"))
        margin(f"RoPE {name} table {maxpos} positions", r)
    q, k, v = (torch.zeros(frames, heads, T, 64, device="cuda", dtype=BF16) for _ in range(3))
    ops.qkv_proj(a, w, bias, *ln, q, k, v, ntok=T, T=T, nspecial=5, wp=wp, rope_cos=cos, rope_sin=sin, block_n=bn)
    qscale = float(torch.tensor((1.0 / math.sqrt(64.0)) * math.log2(math.e), dtype=F32))
    refs, bnds = R.qkv_ref(a, w, bias, heads, T, qscale, ln=ln, rope=(cos, sin, _positions(M, T, 5, wp)))
    torch.cuda.synchronize()
    for name, out, ref, bnd in zip("qkv", (q, k, v), refs, bnds):
        r, f = R.check_rounded(out, ref, bnd, BF16, f"QKV {name} C={C}", ("seq", "head", "tok", "col"))
        margin(f"QKV {name} C={C} {hp}x{wp}", r)


@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("outc,act", [(2, 0), (4, 1)])
def test_headtail_per_element(outc, act, dtype):
    """EPI_HEADTAIL (gemm_kernel<32, EPI_HEADTAIL>): 3x3 conv 128 -> 32 + ReLU + 1x1 + activations, fp32 outputs, against the bound."""
    ops = ops_module()
    Fr, h, w, Cin = 2, 14, 28, 128
    x = randn(Fr, h + 2, w + 2, Cin, seed=1)
    x[:, 0], x[:, -1], x[:, :, 0], x[:, :, -1] = 0, 0, 0, 0
    xp = x.to(dtype)
    wb = randn(32, 9 * Cin, scale=(9 * Cin) ** -0.5, seed=2, dtype=dtype)
    b1, w2, b2 = randn(32, scale=0.1, seed=3), randn(outc, 32, scale=32 ** -0.5, seed=4), randn(outc, scale=0.1, seed=5)
    preds = torch.zeros(Fr, h, w, outc - 1, device="cuda")
    conf = torch.zeros(Fr, h, w, device="cuda")
    taps = [(ky - 1) * (w + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    ops.gemm(xp.reshape(-1, Cin), wb, taps=taps, epi=ops.L.EPI_HEADTAIL, bias=b1, w2=w2, b2=b2, outc=outc, head_act=act,
             preds=preds, conf=conf, rowmap=ops.L.ROWS_PAD, gh=h, gw=w)
    rp, rc, bp, bc = R.headtail_ref(xp.reshape(-1, Cin), wb, taps, b1, w2, b2, act, Fr, h, w)
    torch.cuda.synchronize()
    r1 = R.check_bound(preds, rp, bp, "HEADTAIL preds", ("frame", "y", "x", "c"))
    r2 = R.check_bound(conf, rc, bc, "HEADTAIL conf", ("frame", "y", "x"))
    margin(f"HEADTAIL outc={outc} act={act} {dtype}", max(r1, r2))


# ----------------------------------------------------------------------------------------------- attention
def _attn_shape(path, sms):
    """(batch, heads, nq, nkv, scratch) that takes `path` on this device."""
    if path == "plain":
        return 1, 2, 300, 300, False
    if path == "persistent":
        return 2, 16, 1374, 1374, False
    if path == "cross_plain":
        return 2, 3, 300, 1374, False
    if path == "cross_persistent":
        return 4, 16, 700, 1374, False
    if path in REAL_SHAPES:
        B, H, n = REAL_SHAPES[path]
        return B, H, n, n, True
    parts = int(path[-1])
    n = 24 * 128 + 37                                   # 25 KV tiles (>= 24: split allowed), ragged last tile
    for h in range(1, 400):
        if R.attention_path(1, h, n, n, sms, True) == ("split", parts):
            return 1, h, n, n, True
    pytest.skip(f"no head count splits in {parts} parts on {sms} SMs")


PATHS = ["plain", "persistent", "split2", "split3", "split4", "cross_plain", "cross_persistent"]
# (batch, heads, tokens) as the model launches attention for 294-, 392- and 882-pixel-high inputs of a 518-pixel width with 5, 10
# and 3 views: frame attention over each view's T = hp * wp + 5 tokens, global attention over a scene's S * T.  They leave ragged
# last tiles other than the 518 x 518 ones, and whichever path this device's launch rule picks for them is the one tested.
REAL_SHAPES = {"frame 294x518": (5, 16, 782), "global 294x518": (1, 16, 3910), "frame 392x518": (10, 16, 1041),
               "global 392x518": (1, 16, 10410), "frame 882x518": (3, 16, 2336), "global 882x518": (1, 16, 7008)}


def _run_attention(q, k, v, B, H, nq, nkv, scratch):
    """ovg_attention on the device; returns (out, launches, scratch bytes written)."""
    ops, L = ops_module(), lib_module()
    out = torch.zeros(B, nq, H * 64, device="cuda", dtype=BF16)
    s = None
    if scratch:
        s = ops.attention_scratch("cuda")
        s.fill_(0xFF)                                    # all-ones words: NaN as fp32
    n0 = L.lib().ovg_launch_count()
    ops.attention(q.cuda(), k.cuda(), v.cuda(), out, B, H, nq, nkv, scratch=s)
    launches = L.lib().ovg_launch_count() - n0
    torch.cuda.synchronize()
    written = 0
    if scratch:
        w = s[:(s.numel() - 256) // 4 * 4].view(torch.int32) != -1
        written = int(w.nonzero().max()) * 4 + 4 if bool(w.any()) else 0
    return out, launches, written


def _check_path(path, sms, B, H, nq, nkv, scratch, launches, written):
    kind, parts = R.attention_path(B, H, nq, nkv, sms, scratch)
    if path not in REAL_SHAPES:
        assert kind == {"plain": "plain", "persistent": "persistent", "cross_plain": "plain", "cross_persistent": "persistent"}.get(
            path, "split")
    assert launches == (2 if kind == "split" else 1), launches
    if kind == "split":      # exactly the partial results of `parts` KV ranges per tail tile were written
        assert written == R.split_scratch_bytes(B, H, nq, sms, parts), (written, parts)
    print(f"attention {path}: B={B} H={H} nq={nq} nkv={nkv} -> {kind}, {parts} part(s), {launches} launch(es)")


@pytest.mark.parametrize("path", PATHS)
def test_attention_onehot_exact(path, sms):
    """Each query's weight on one key: out = v[target] bit for bit on every path."""
    B, H, nq, nkv, scratch = _attn_shape(path, sms)
    q, k, v, exp = R.onehot_case(B, H, nq, nkv, seed=1)
    out, launches, written = _run_attention(q, k, v, B, H, nq, nkv, scratch)
    _check_path(path, sms, B, H, nq, nkv, scratch, launches, written)
    bad = (out.cpu() != exp).any(-1).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} rows differ, first (batch, row) {tuple(bad[0].tolist())}"


@pytest.mark.parametrize("path", PATHS)
def test_attention_rounding_rows(path, sms):
    """l must sum the unrounded probabilities: on rows where every bf16 rounding of P goes the same way, >= 99 % of the outputs
    equal the fp64 result rounded once."""
    B, H, nq, nkv, scratch = _attn_shape(path, sms)
    if nq != nkv:
        pytest.skip("self-attention construction")
    q, k, v, ref = R.rounding_case(B, H, nq, seed=2)
    out, *_ = _run_attention(q, k, v, B, H, nq, nkv, scratch)
    ref, bound = R.attention_ref(q.cuda(), k.cuda(), v.cuda())
    r, f = R.check_rounded(out, ref, bound, BF16, f"attention rounding rows ({path})", ("batch", "row", "col"))
    margin(f"attention rounding rows {path}", r)


@pytest.mark.parametrize("n", [1, 33, 127, 128, 129, 1374, 9000] + sorted(n for *_, n in REAL_SHAPES.values()))
def test_attention_uniform_rows_exact(n, sms):
    """Every probability exactly 1: out = the column mean of v, bit for bit (a key the mask should drop would take nearly all the
    weight).  9000 keys with scratch also run the split path where this device's cost rule splits them.  The frame and global
    lengths of the non-square inputs (REAL_SHAPES) run at the model's batch and 16 heads."""
    B, H = next(((b, h) for b, h, m in REAL_SHAPES.values() if m == n), (1, 2))
    q, k, v, exp = R.uniform_case(B, H, n, seed=n)
    out, launches, _ = _run_attention(q, k, v, B, H, n, n, True)
    print(f"uniform B={B} H={H} n={n}: {R.attention_path(B, H, n, n, sms, True)}, {launches} launch(es)")
    bad = (out.cpu() != exp).any(-1).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} rows differ, first (batch, row) {tuple(bad[0].tolist())}"


def _rand_attn(B, H, nq, nkv, kind, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, H, nq, 64, generator=g, dtype=F64) * (math.log2(math.e) / 8)
    k = torch.randn(B, H, nkv, 64, generator=g, dtype=F64)
    if kind == "peaky":
        q *= 1.5
        k *= torch.linspace(0.2, 6.0, nkv, dtype=F64)[None, None, :, None]
    elif kind == "spike":                        # one late key whose logit exceeds the others by > 2^7 (log2 units)
        q = q * 0.3 + 2.0
        k = k * 0.3
        k[:, :, nkv - 3] = 3.0
    v = torch.randn(B, H, nkv, 64, generator=g, dtype=F64)
    return q.to(BF16), k.to(BF16), v.to(BF16)


@pytest.mark.parametrize("kind", ["random", "peaky", "spike"])
@pytest.mark.parametrize("path", PATHS + list(REAL_SHAPES))
def test_attention_per_element(path, kind, sms):
    """Random, peaky and late-spike inputs within the per-element bound on every path and at the frame and global shapes of
    the non-square inputs; the split result agrees with the unsplit one within the bound, and repeated runs are bit-identical."""
    B, H, nq, nkv, scratch = _attn_shape(path, sms)
    q, k, v = _rand_attn(B, H, nq, nkv, kind, seed=3)
    out, launches, written = _run_attention(q, k, v, B, H, nq, nkv, scratch)
    _check_path(path, sms, B, H, nq, nkv, scratch, launches, written)
    ref, bound = R.attention_ref(q.cuda(), k.cuda(), v.cuda())
    r = R.check_bound(out, ref, bound, f"attention {kind} ({path})", ("batch", "row", "col"))
    margin(f"attention {kind} {path}", r)
    again, *_ = _run_attention(q, k, v, B, H, nq, nkv, scratch)
    assert torch.equal(out, again)
    if scratch:
        plain, *_ = _run_attention(q, k, v, B, H, nq, nkv, False)
        R.check_bound(plain, ref, bound, f"attention {kind} unsplit", ("batch", "row", "col"))
        rr = R.check_bound(out, plain.double(), 2 * bound, f"attention {kind} split vs unsplit", ("batch", "row", "col"))
        margin(f"attention {kind} split vs unsplit (2x bound)", rr)


# ----------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("C", [128, 384, 1024, 2048])
@pytest.mark.parametrize("in_dtype", [F32, BF16])
@pytest.mark.parametrize("out_dtype", [BF16, F32, F16])
def test_layernorm_per_element(C, in_dtype, out_dtype):
    """Rows with a common offset of 1000 x their spread, near-constant rows where eps dominates, ordinary rows; strided input and
    output (ld > C, sentinels in the gap) and the row gather that drops special tokens."""
    ops = ops_module()
    g = torch.Generator().manual_seed(C)
    rows = 6 * 21
    x = torch.randn(rows, C, generator=g, dtype=F64) * 3 + 0.5
    x[:40] += 1e3 * torch.randn(40, 1, generator=g, dtype=F64) * 3
    x[40:60] = 0.25 + 1e-4 * torch.randn(20, C, generator=g, dtype=F64)
    w, b = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    xin = torch.full((rows, C + 64), 77.0, dtype=in_dtype)
    xin[:, :C] = x.to(in_dtype)
    xin = xin.cuda()
    for gather in (False, True):
        orows = 6 * 16 if gather else rows
        src = xin[:, :C].double().cpu()
        if gather:
            src = src.reshape(6, 21, C)[:, 5:].reshape(orows, C)
        fill = -3.0
        obuf = torch.full((orows, C + 32), fill, device="cuda", dtype=out_dtype)
        kw = dict(grp_out=16, grp_in=21, grp_off=5) if gather else {}
        ops.layernorm(xin[:, :C], obuf[:, :C], w.cuda(), b.cuda(), 1e-5, **kw)
        ref, bound = R.layernorm_ref(src, w, b, 1e-5, out_dtype)
        torch.cuda.synchronize()
        r = R.check_bound(obuf[:, :C], ref, bound, f"LayerNorm C={C}", ("row", "col"))
        assert (obuf[:, C:] == fill).all()
        margin(f"LayerNorm C={C} {in_dtype}->{out_dtype} gather={gather}", r)


# ----------------------------------------------------------------------------------------------- camera head
def _camera_model(embed_dim, heads, trunk=2, seed=0):
    from omnivggt_official_b200 import OmniVGGT
    m = OmniVGGT(img_size=56, embed_dim=embed_dim, depth=1, patch_embed="conv", dpt_features=128,
                 dpt_out_channels=(64, 128, 256, 256), dpt_layers=(0, 0, 0, 0), camera_heads=heads, camera_trunk_depth=trunk,
                 init_seed=None).cuda()
    m.randomize_(seed=seed)
    m.point_head = None
    m.depth_head = None
    return m


@pytest.mark.parametrize("embed_dim,heads", [(128, 8), (128, 4), (128, 2), (128, 1), (1024, 16)])
def test_camera_head_against_fp64(embed_dim, heads):
    """model.camera_head for head_dim 32, 64, 128, 256 (D = 256) and the full width (D = 2048, 16 heads), S in {1, 3, 24},
    B in {1, 2}, 4 iterations, against the fp64 restatement with the runtime's bf16 roundings; scene b of a B = 2 call equals that
    scene run alone, bit for bit."""
    m = _camera_model(embed_dim, heads, trunk=2 if embed_dim == 128 else 4)
    eng = m.engine()
    D = 2 * embed_dim
    worst = 0.0
    for S in (1, 3, 24):
        tok = randn(2, S, 1, D, seed=S)
        out = torch.stack(m.camera_head([tok], num_iterations=4))            # [4, B, S, 9]
        ref = R.camera_ref(eng.cam, tok.reshape(2 * S, D), 2, S, heads)
        e = R.camera_error(out.reshape(4, 2 * S, 9), ref)
        print(f"camera D={D} heads={heads} S={S}: error {e:.2e} of max |pose|")
        assert e <= R.CAM_TOL, e
        worst = max(worst, e)
        for bi in range(2):
            alone = torch.stack(m.camera_head([tok[bi:bi + 1]], num_iterations=4))
            assert torch.equal(alone[:, 0], out[:, bi]), (S, bi)
    margin(f"camera head D={D} heads={heads} (error / CAM_TOL)", worst / R.CAM_TOL)
