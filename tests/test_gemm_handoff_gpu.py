"""The GEMM's hand-off of finished accumulator tiles from its wgmma warpgroups to its epilogue warpgroup, over many tiles per CTA.

gemm_kernel stages each tile's accumulators in one shared-memory tile that the epilogue warpgroup reads while the wgmma warpgroups
already run the next tile's K loop.  A slip in that hand-off shows up only when a CTA runs several tiles in a row, so every test
here gives each CTA at least three tiles (derived from this device's SM count), with a total that is not a multiple of the grid,
for every epilogue kind.  K = 64 makes the K loop shorter than the epilogue (the wgmma warpgroups wait for the staging tile to be
free); K >= 512 makes it longer.  Integer operands make the results exact, so the tests assert bit equality, except for GELU and
the QKV LayerNorm + RoPE, which are held to the element-wise bounds of oracle/kernel_ref.py."""
import math
import os
import sys

import pytest
import torch

from oracle import kernel_ref as R

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_bounds_gpu import _guarded, _guards_ok, _margin, _positions, _randn  # noqa: E402

pytestmark = pytest.mark.gpu

BF16, F16, F64 = torch.bfloat16, torch.float16, torch.float64
FILL = -3.0


def _ops():
    from omnivggt_official_b200 import ops
    return ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _m_tiles(sms, n_tiles, per_cta=3):
    """Row tiles for at least `per_cta` tiles per CTA (the grid is min(tiles, SMs) CTAs) and a tile count that is not a multiple
    of the grid, so that the CTAs end on different tiles."""
    m = -(-(per_cta * sms + 1) // n_tiles)
    while (m * n_tiles) % sms == 0:
        m += 1
    return m


def _int_gpu(rows, n, K, seed):
    a, b = R.int_operands(rows, n, K, seed=seed)
    return a.cuda(), b.cuda()


@pytest.mark.parametrize("K", [64, 1024])
@pytest.mark.parametrize("dtype", [BF16, F16])
@pytest.mark.parametrize("bn", [64, 128])
def test_handoff_bf16_exact(bn, dtype, K, sms):
    """EPI_BF16, identity rows, ragged last row tile, guards around the output."""
    ops = _ops()
    N = 256
    M = 128 * _m_tiles(sms, N // bn) - 37
    a, b = _int_gpu(M, N, K, seed=K + bn)
    bias = torch.randint(-300, 300, (N,)).double().cuda()
    buf, flat = _guarded(M * N, dtype, FILL)
    ops.gemm(a.to(dtype), b.to(dtype), epi=ops.L.EPI_BF16, bias=bias.float(), out=flat, ldo=N, block_n=bn)
    acc, _ = R.gemm_acc(a, b)
    exp = R.round_to(acc + bias[None], dtype)
    torch.cuda.synchronize()
    got = flat.view(M, N).double()
    bad = (got != exp).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} mismatches, first at (row, col) {tuple(bad[0].tolist())}"
    assert _guards_ok(buf, FILL)


def test_handoff_gelu_per_element(sms):
    """EPI_BF16 with the exact-erf GELU, fc1-shaped (N = 1024, K = 1024) at 128 x 128 tiles."""
    ops = _ops()
    N, K = 1024, 1024
    M = 128 * _m_tiles(sms, N // 128) - 5
    a = _randn(M, K, seed=1, dtype=BF16)
    w = _randn(N, K, scale=K ** -0.5, seed=2, dtype=BF16)
    bias = _randn(N, seed=3)
    out = torch.empty(M, N, device="cuda", dtype=BF16)
    ops.gemm(a, w, epi=ops.L.EPI_BF16, bias=bias, act=ops.L.ACT_GELU, out=out, ldo=N, block_n=128)
    ref, bound = R.linear_ref(a, w, bias, act="gelu", out_dtype=BF16)
    torch.cuda.synchronize()
    r, f = R.check_rounded(out, ref, bound, BF16, f"GEMM+GELU {M}x{N}x{K}", ("row", "col"))
    _margin(f"handoff GEMM+GELU {M}x{N}x{K}", r)


@pytest.mark.parametrize("K", [64, 512])
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("scatter", [False, True])
def test_handoff_resid_exact(scatter, bn, K, sms):
    """EPI_RESID: x[row] += gamma (acc + bias) in fp32 with power-of-two gamma, rows direct or scattered through row_index."""
    ops = _ops()
    N = 256
    M = 128 * _m_tiles(sms, N // bn) - 11
    a, b = _int_gpu(M, N, K, seed=M + K)
    g = torch.Generator().manual_seed(N + bn)
    bias = torch.randint(-200, 200, (N,), generator=g).double()
    gamma = torch.tensor([0.5, 2.0, -0.25, 1.0])[torch.randint(0, 4, (N,), generator=g)].double()
    x0 = torch.randint(-1000, 1000, (M, N), generator=g).double()
    perm = torch.randperm(M, generator=g)
    x = x0.float().cuda()
    ops.linear_resid(a.to(BF16), b.to(BF16), bias.float().cuda(), gamma.float().cuda(), x,
                     row_index=perm.int().cuda() if scatter else None, block_n=bn)
    acc, _ = R.gemm_acc(a, b)
    exp = x0.cuda()
    upd = gamma.cuda() * (acc + bias.cuda())
    if scatter:
        exp[perm.cuda()] += upd
    else:
        exp += upd
    torch.cuda.synchronize()
    assert torch.equal(x.double(), exp)


@pytest.mark.parametrize("bn", [64, 128])
def test_handoff_qkv_norm_rope(bn, sms):
    """EPI_QKV with the q / k LayerNorm(64) and 2-D RoPE at the aggregator's token layout (37 x 37 patches + 5 special tokens)."""
    ops = _ops()
    C, hp, wp = 256, 37, 37
    heads, T = C // 64, hp * wp + 5
    frames = -(-128 * _m_tiles(sms, 3 * C // bn) // T)
    M = frames * T
    assert -(-M // 128) * (3 * C // bn) >= 3 * sms
    a = _randn(M, C, seed=1, dtype=BF16)
    w = _randn(3 * C, C, scale=C ** -0.5, seed=2, dtype=BF16)
    bias = _randn(3 * C, scale=0.1, seed=3)
    ln = [1 + 0.1 * _randn(64, seed=4), 0.1 * _randn(64, seed=5), 1 + 0.1 * _randn(64, seed=6), 0.1 * _randn(64, seed=7)]
    cos, sin = ops.rope_tables(max(hp, wp) + 1, "cuda")
    q, k, v = (torch.zeros(frames, heads, T, 64, device="cuda", dtype=BF16) for _ in range(3))
    ops.qkv_proj(a, w, bias, *ln, q, k, v, ntok=T, T=T, nspecial=5, wp=wp, rope_cos=cos, rope_sin=sin, block_n=bn)
    qscale = float(torch.tensor((1.0 / math.sqrt(64.0)) * math.log2(math.e), dtype=torch.float32))
    refs, bnds = R.qkv_ref(a, w, bias, heads, T, qscale, ln=ln, rope=(cos, sin, _positions(M, T, 5, wp)))
    torch.cuda.synchronize()
    for name, out, ref, bnd in zip("qkv", (q, k, v), refs, bnds):
        r, f = R.check_rounded(out, ref, bnd, BF16, f"QKV {name} bn={bn}", ("seq", "head", "tok", "col"))
        _margin(f"handoff QKV {name} bn={bn}", r)


@pytest.mark.parametrize("dtype", [BF16, F16])
def test_handoff_pad_taps_skips_exact(dtype, sms):
    """RM_PAD, a 3 x 3 conv as 9 row-shifted taps over a zero-bordered grid with two skips and ReLU: border rows written as zeros,
    interior = relu(taps + bias + skips)."""
    ops = _ops()
    gh, gw, Cin, N, bn = 78, 78, 64, 128, 64
    per_frame = (gh + 2) * (gw + 2)
    F = -(-128 * _m_tiles(sms, N // bn) // per_frame)
    rows = F * per_frame
    assert -(-rows // 128) * (N // bn) >= 3 * sms
    taps = [(ky - 1) * (gw + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    g = torch.Generator().manual_seed(12)
    a = torch.randint(-8, 9, (rows, Cin), generator=g).double().cuda()
    b = torch.randint(-8, 9, (N, 9 * Cin), generator=g).double().cuda()
    s1, s2 = (torch.randint(-64, 65, (rows, N), generator=g).double().cuda() for _ in range(2))
    bias = torch.randint(-200, 200, (N,), generator=g).double().cuda()
    buf, flat = _guarded(rows * N, dtype, FILL)
    ops.gemm(a.to(dtype), b.to(dtype), taps=taps, epi=ops.L.EPI_BF16, bias=bias.float(), act=ops.L.ACT_RELU, out=flat, ldo=N,
             skip1=s1.to(dtype), skip2=s2.to(dtype), rowmap=ops.L.ROWS_PAD, gh=gh, gw=gw, block_n=bn)
    acc, _ = R.gemm_acc(a, b, taps)
    exp = R.round_to((acc + bias[None] + s1 + s2).clamp(min=0), dtype).reshape(F, gh + 2, gw + 2, N)
    exp[:, 0], exp[:, -1], exp[:, :, 0], exp[:, :, -1] = 0.0, 0.0, 0.0, 0.0
    torch.cuda.synchronize()
    assert torch.equal(flat.view(F, gh + 2, gw + 2, N).double(), exp) and _guards_ok(buf, FILL)
