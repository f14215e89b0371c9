"""The GEMM's residual epilogue (EPI_RESID), which walks each accumulator tile row by row across a warp: BN / 4 lanes per row,
one float4 each, several rows in flight.

Every block_n runs (32, 64 and 128: 8, 16 and 32 lanes per row), with N a multiple of block_n and not (the last column tile
half outside N), a single row tile and many tiles per CTA with a ragged last row tile, and rows direct or scattered through
row_index.  x has guard rows above and below that must stay untouched.  Integer operands and power-of-two gamma make every
value exact, so the tests assert bit equality."""
import pytest
import torch

from oracle import kernel_ref as R

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
GUARD_ROWS = 128


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("rows", ["one_tile", "many_tiles"])
@pytest.mark.parametrize("N", [256, 160])
@pytest.mark.parametrize("bn", [32, 64, 128])
@pytest.mark.parametrize("scatter", [False, True])
def test_resid_rows_exact(scatter, bn, N, rows, sms):
    from omnivggt_official_b200 import ops
    K = 192
    n_tiles = -(-N // bn)
    M = 77 if rows == "one_tile" else 128 * -(-(3 * sms + 1) // n_tiles) - 11
    g = torch.Generator().manual_seed(N + bn + M)
    a, b = R.int_operands(M, N, K, seed=M + K)
    a, b = a.cuda(), b.cuda()
    bias = torch.randint(-200, 200, (N,), generator=g).double()
    gamma = torch.tensor([0.5, 2.0, -0.25, 1.0])[torch.randint(0, 4, (N,), generator=g)].double()
    x0 = torch.randint(-1000, 1000, (M + 2 * GUARD_ROWS, N), generator=g).double()
    perm = torch.randperm(M, generator=g)
    xall = x0.float().cuda()
    x = xall[GUARD_ROWS:GUARD_ROWS + M]
    ops.linear_resid(a.to(BF16), b.to(BF16), bias.float().cuda(), gamma.float().cuda(), x,
                     row_index=perm.int().cuda() if scatter else None, block_n=bn)
    acc, _ = R.gemm_acc(a, b)
    exp = x0.cuda()
    upd = gamma.cuda() * (acc + bias.cuda())
    if scatter:
        exp[GUARD_ROWS + perm.cuda()] += upd
    else:
        exp[GUARD_ROWS:GUARD_ROWS + M] += upd
    torch.cuda.synchronize()
    bad = (xall.double() != exp).nonzero()
    assert bad.numel() == 0, f"{bad.shape[0]} mismatches, first at (row incl. guard, col) {tuple(bad[0].tolist())}"
