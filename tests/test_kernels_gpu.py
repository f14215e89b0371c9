"""Kernel-level parity (GPU): every libovg entry point against a plain PyTorch fp32 reference of the same op, through
the C ABI.  Tolerances (stated per test) are for bf16 operands / fp32 accumulation."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32


def _ops():
    from omnivggt_official_b200 import ops
    return ops


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def randn(*s, scale=1.0, seed=0, dtype=F32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*s, generator=g, device="cuda") * scale).to(dtype)


# ----------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K,bn", [(128, 64, 64, 0), (300, 256, 128, 0), (1000, 384, 192, 128), (2748, 3072, 1024, 256),
                                      (515, 1024, 4096, 128), (77, 96, 392, 64),
                                      # block_n above 128 (the widest tile) runs as 128
                                      (2748, 3072, 1024, 512), (515, 1024, 4096, 512), (300, 256, 128, 512), (129, 512, 64, 512),
                                      (10992, 1024, 1024, 512),
                                      # many tiles with a short last wave
                                      (5000, 1024, 128, 512), (4000, 1280, 64, 512), (19000, 256, 64, 512),
                                      (2748, 384, 192, 384), (1500, 128, 2048, 384), (300, 256, 128, 384)])
def test_gemm_bf16_bias_gelu(M, N, K, bn):
    ops = _ops()
    a = randn(M, K, seed=1, dtype=BF16)
    w = randn(N, K, scale=K ** -0.5, seed=2, dtype=BF16)
    bias = randn(N, seed=3)
    out = ops.linear_bf16(a, w, bias, act=ops.L.ACT_GELU, block_n=bn)
    ref = F.gelu(a.float() @ w.float().t() + bias)
    torch.cuda.synchronize()
    assert rel(out, ref) < 6e-3          # bf16 output rounding ~ 2^-9
    out2 = ops.linear_bf16(a, w, None, act=ops.L.ACT_NONE, block_n=bn)
    assert rel(out2, a.float() @ w.float().t()) < 6e-3


@pytest.mark.parametrize("M,N,K,bn", [(5000, 1024, 128, 512), (10992, 1024, 256, 512)])
def test_gemm_resid_split_tail(M, N, K, bn):
    """Residual epilogue (fp32 read-modify-write) over a tile count with a short last wave."""
    ops = _ops()
    a = randn(M, K, seed=1, dtype=BF16)
    w = randn(N, K, scale=K ** -0.5, seed=2, dtype=BF16)
    bias, gamma = randn(N, seed=3), randn(N, seed=4)
    x0 = randn(M, N, seed=5)
    x = x0.clone()
    ops.linear_resid(a, w, bias, gamma, x, block_n=bn)
    ref = x0 + gamma * (a.float() @ w.float().t() + bias)
    assert rel(x, ref) < 1e-5


@pytest.mark.parametrize("bn", [0, 512])
def test_gemm_resid_rowindex(bn):
    ops = _ops()
    M, N, K = 1374 * 2, 1024, 1024
    a = randn(M, K, seed=1, dtype=BF16)
    w = randn(N, K, scale=K ** -0.5, seed=2, dtype=BF16)
    bias, gamma = randn(N, seed=3), randn(N, seed=4)
    x0 = randn(M, N, seed=5)
    x = x0.clone()
    ops.linear_resid(a, w, bias, gamma, x, block_n=bn)
    ref = x0 + gamma * (a.float() @ w.float().t() + bias)
    assert rel(x, ref) < 1e-5 + 2e-3 * 0  # fp32 output: only accumulation-order noise
    # scatter rows
    perm = torch.randperm(M, device="cuda", dtype=torch.int32)
    x = x0.clone()
    ops.linear_resid(a, w, bias, gamma, x, row_index=perm, block_n=bn)
    ref2 = x0.clone()
    ref2[perm.long()] += gamma * (a.float() @ w.float().t() + bias)
    assert rel(x, ref2) < 1e-5


def _rope_ref(t, pos, base=100.0):
    # t [Bx,H,N,64] fp32, pos [Bx,N,2]
    half = 32
    inv = 1.0 / (base ** (torch.arange(0, half, 2, device=t.device).float() / half))

    def one(z, p):
        ang = p[:, None, :, None].float() * inv
        c, s = ang.cos(), ang.sin()
        a, b = z[..., :16], z[..., 16:]
        return torch.cat([a * c - b * s, b * c + a * s], -1)

    return torch.cat([one(t[..., :32], pos[..., 0]), one(t[..., 32:], pos[..., 1])], -1)


@pytest.mark.parametrize("C,frames,hp,wp,S,bn", [(128, 3, 4, 4, 3, 0), (1024, 2, 37, 37, 2, 0), (256, 4, 3, 5, 2, 0),
                                                 (1024, 2, 37, 37, 2, 512), (128, 3, 4, 4, 3, 512),
                                                 (1024, 2, 29, 30, 2, 512)])   # 84 tiles: split last wave
def test_gemm_qkv_epilogue(C, frames, hp, wp, S, bn):
    """QKV linear + q/k LayerNorm(64) + 2-D RoPE + head-major layout vs reference formulas
    (layers/attention.py:52-58, layers/rope.py:154-188)."""
    ops = _ops()
    heads, T = C // 64, hp * wp + 5
    M = frames * T
    a = randn(M, C, seed=1, dtype=BF16)
    w = randn(3 * C, C, scale=C ** -0.5, seed=2, dtype=BF16)
    bias = randn(3 * C, scale=0.1, seed=3)
    qn_w, qn_b, kn_w, kn_b = 1 + 0.1 * randn(64, seed=4), 0.1 * randn(64, seed=5), 1 + 0.1 * randn(64, seed=6), 0.1 * randn(64, seed=7)
    cos, sin = ops.rope_tables(max(hp, wp) + 1, "cuda")
    for ntok in (T, S * T):   # frame-wise and global views of the same rows
        if M % ntok:
            continue
        nb = M // ntok
        # outputs carved out of sentinel-filled buffers: bulk stores that straddle a sequence boundary must not touch
        # anything outside [nb, heads, ntok, 64]
        guard = 4096
        bufs = [torch.full((guard + nb * heads * ntok * 64 + guard,), 7.0, device="cuda", dtype=BF16) for _ in range(3)]
        q, k, v = (b[guard:-guard].view(nb, heads, ntok, 64) for b in bufs)
        for t in (q, k, v):
            t.zero_()
        ops.qkv_proj(a, w, bias, qn_w, qn_b, kn_w, kn_b, q, k, v, ntok=ntok, T=T, nspecial=5, wp=wp, rope_cos=cos, rope_sin=sin, block_n=bn)
        qkv = (a.float() @ w.float().t() + bias).reshape(nb, ntok, 3, heads, 64).permute(2, 0, 3, 1, 4)
        yy, xx = torch.meshgrid(torch.arange(hp, device="cuda"), torch.arange(wp, device="cuda"), indexing="ij")
        pos = torch.cat([torch.zeros(5, 2, device="cuda", dtype=torch.long), torch.stack([yy.reshape(-1), xx.reshape(-1)], -1) + 1])
        pos = pos[None].expand(frames, -1, -1).reshape(nb, ntok, 2)
        qr = _rope_ref(F.layer_norm(qkv[0], (64,), qn_w, qn_b, 1e-5), pos) * (math.log2(math.e) / 8.0)
        kr = _rope_ref(F.layer_norm(qkv[1], (64,), kn_w, kn_b, 1e-5), pos)
        torch.cuda.synchronize()
        assert rel(q, qr) < 6e-3 and rel(k, kr) < 6e-3 and rel(v, qkv[2]) < 6e-3
        for b in bufs:
            assert (b[:guard] == 7.0).all() and (b[-guard:] == 7.0).all()


# ----------------------------------------------------------------------------------------------- attention
@pytest.mark.parametrize("batch,heads,n", [(1, 1, 128), (1, 2, 256), (2, 2, 200), (3, 2, 1374), (1, 16, 2 * 1374), (1, 4, 700), (1, 2, 1), (2, 1, 33),
                                           (1, 3, 64), (1, 2, 129), (1, 2, 257), (1, 2, 320), (2, 3, 385)])
def test_attention(batch, heads, n):
    """vs softmax(q k^T / 8) v in fp32 (layers/attention.py:61-66).  bf16 P and bf16 output: rel-L2 < 1e-2."""
    ops = _ops()
    q = randn(batch, heads, n, 64, seed=1)
    k = randn(batch, heads, n, 64, seed=2)
    v = randn(batch, heads, n, 64, seed=3)
    qs = (q * (math.log2(math.e) / 8.0)).to(BF16)
    kb, vb = k.to(BF16), v.to(BF16)
    out = torch.zeros(batch, n, heads * 64, device="cuda", dtype=BF16)
    ops.attention(qs, kb, vb, out, batch, heads, n)
    s = (qs.float() * math.log(2.0)) @ kb.float().transpose(-1, -2)
    ref = (s.softmax(-1) @ vb.float()).transpose(1, 2).reshape(batch, n, heads * 64)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    assert rel(out, ref) < 1e-2, rel(out, ref)


def _sdpa_fp32_chunked(qs, kb, vb, qchunk=4096):
    """softmax(q k^T) v in fp32, one head and `qchunk` query rows at a time (the score matrix of the 24-view global
    attention is 16 x 32 976^2 fp32 = 70 GB in one piece)."""
    batch, heads, n, _ = qs.shape
    out = torch.empty(batch, n, heads * 64, device=qs.device, dtype=F32)
    ln2 = math.log(2.0)
    for b in range(batch):
        for h in range(heads):
            kf, vf = kb[b, h].float(), vb[b, h].float()
            for i0 in range(0, n, qchunk):
                s = (qs[b, h, i0:i0 + qchunk].float() * ln2) @ kf.t()
                out[b, i0:i0 + qchunk, h * 64:(h + 1) * 64] = s.softmax(-1) @ vf
    return out


@pytest.mark.parametrize("heads,n", [(16, 8 * 1374), (16, 24 * 1374)])
def test_attention_global_sizes_of_baseline_configs(heads, n):
    """BASELINE.json configs[1] / configs[4]: the global attention of 8 views (L = 10 992, 172 KV steps) and of 24 views
    (L = 32 976, 516 KV steps), 16 heads, against fp32 SDPA (reference layers/attention.py:61-66) -- same 1e-2 bar as the
    small shapes; the long accumulation (fp32 O / l in registers, online rescaling) is what is under test."""
    ops = _ops()
    q = randn(1, heads, n, 64, seed=1)
    k = randn(1, heads, n, 64, seed=2)
    v = randn(1, heads, n, 64, seed=3)
    qs = (q * (math.log2(math.e) / 8.0)).to(BF16)
    kb, vb = k.to(BF16), v.to(BF16)
    del q, k, v
    out = torch.zeros(1, n, heads * 64, device="cuda", dtype=BF16)
    ops.attention(qs, kb, vb, out, 1, heads, n)
    ref = _sdpa_fp32_chunked(qs, kb, vb)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    e = rel(out, ref)
    print(f"attention n={n}: rel-L2 {e:.3e}")
    assert e < 1e-2, e
    out2 = torch.zeros_like(out)
    ops.attention(qs, kb, vb, out2, 1, heads, n)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)          # run-to-run bit-identical (no atomics, no ordering races)
    # with scratch the tiles of the last CTA wave are split over the keys and merged (ovg_attention scratch): same bar, deterministic
    scratch = ops.attention_scratch("cuda")
    out3, out4 = torch.zeros_like(out), torch.zeros_like(out)
    ops.attention(qs, kb, vb, out3, 1, heads, n, scratch=scratch)
    ops.attention(qs, kb, vb, out4, 1, heads, n, scratch=scratch)
    torch.cuda.synchronize()
    e3 = rel(out3, ref)
    print(f"attention n={n} (split tail): rel-L2 {e3:.3e}, vs unsplit {rel(out3, out):.3e}")
    assert e3 < 1e-2 and torch.equal(out3, out4) and rel(out3, out) < 4e-3


@pytest.mark.parametrize("batch,heads,n", [(1, 16, 4 * 1374), (2, 16, 4 * 1374), (1, 7, 9000)])
def test_attention_split_tail_shapes(batch, heads, n):
    """Attention with scratch at other tile counts, ragged last KV tile, peaky rows.  On an H100 SXM (132 resident CTAs, one per SM)
    688 tiles leave a last wave of 28 tiles, split in 3 parts; 1 376 tiles over two batch entries leave 56, split in 2; 497 tiles leave
    101, which the cost rule does not split, so that case checks the unsplit path with scratch given.  test_kernel_bounds_gpu.py
    asserts which path each of its shapes takes on the device it runs on."""
    ops = _ops()
    q = randn(batch, heads, n, 64, seed=1) * 1.5
    k = randn(batch, heads, n, 64, seed=2)
    v = randn(batch, heads, n, 64, seed=3)
    k[:, :, n - 3] *= 6.0                    # a late dominant key: the parts end on very different references
    qs = (q * (math.log2(math.e) / 8.0)).to(BF16)
    kb, vb = k.to(BF16), v.to(BF16)
    del q, k, v
    scratch = ops.attention_scratch("cuda")
    out = torch.zeros(batch, n, heads * 64, device="cuda", dtype=BF16)
    ops.attention(qs, kb, vb, out, batch, heads, n, scratch=scratch)
    ref = _sdpa_fp32_chunked(qs, kb, vb)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    assert rel(out, ref) < 1e-2, rel(out, ref)


def test_attention_peaky_rows_rescale():
    """Large, growing logits force the lazy-rescale path (running max grows by > 8 between KV tiles)."""
    ops = _ops()
    batch, heads, n = 1, 2, 1024
    q = randn(batch, heads, n, 64, seed=1)
    k = randn(batch, heads, n, 64, seed=2) * torch.linspace(0.2, 6.0, n, device="cuda")[None, None, :, None]
    v = randn(batch, heads, n, 64, seed=3)
    qs, kb, vb = q.to(BF16), k.to(BF16), v.to(BF16)
    out = torch.zeros(batch, n, heads * 64, device="cuda", dtype=BF16)
    ops.attention(qs, kb, vb, out, batch, heads, n)
    s = (qs.float() * math.log(2.0)) @ kb.float().transpose(-1, -2)
    ref = (s.softmax(-1) @ vb.float()).transpose(1, 2).reshape(batch, n, heads * 64)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    assert rel(out, ref) < 1.5e-2, rel(out, ref)


@pytest.mark.parametrize("spike_at", [130, 650, 699])
def test_attention_late_spike_overflow(spike_at):
    """One key far down the sequence whose logit exceeds everything before it by > 2^128: exp2 against the previous
    maximum would overflow, the kernel must rescale O / l to the new maximum (and keep earlier / later steps exact)."""
    ops = _ops()
    batch, heads, n = 1, 2, 700
    q = randn(batch, heads, n, 64, seed=1) * 0.3 + 2.0
    k = randn(batch, heads, n, 64, seed=2) * 0.3
    k[:, :, spike_at, :] = 3.0                      # q . k ~ 3 * 128 = 384 (log2 units: q is used unscaled)
    k[:, 1, 5, :] = 1.0                             # head 1 additionally has a moderate early peak
    v = randn(batch, heads, n, 64, seed=3)
    qs, kb, vb = q.to(BF16), k.to(BF16), v.to(BF16)
    out = torch.zeros(batch, n, heads * 64, device="cuda", dtype=BF16)
    ops.attention(qs, kb, vb, out, batch, heads, n)
    s = (qs.double() * math.log(2.0)) @ kb.double().transpose(-1, -2)
    ref = (s.softmax(-1) @ vb.double()).transpose(1, 2).reshape(batch, n, heads * 64).float()
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    assert rel(out, ref) < 1.5e-2, rel(out, ref)


# ----------------------------------------------------------------------------------------------- LayerNorm & co
@pytest.mark.parametrize("C", [128, 256, 1024, 2048])
def test_layernorm(C):
    ops = _ops()
    x = randn(777, C, seed=1) * 3 + 0.5
    w, b = 1 + 0.1 * randn(C, seed=2), 0.1 * randn(C, seed=3)
    out = torch.empty(777, C, device="cuda", dtype=BF16)
    ops.layernorm(x, out, w, b, 1e-5)
    assert rel(out, F.layer_norm(x, (C,), w, b, 1e-5)) < 4e-3
    # bf16 input, no affine, row gather that drops 5 special tokens per frame
    T, P = 21, 16
    xb = randn(4 * T, C, seed=4, dtype=BF16)
    out2 = torch.empty(4 * P, C, device="cuda", dtype=BF16)
    ops.layernorm(xb, out2, None, None, 1e-5, grp_out=P, grp_in=T, grp_off=5)
    ref = F.layer_norm(xb.float().reshape(4, T, C)[:, 5:], (C,), None, None, 1e-5).reshape(4 * P, C)
    assert rel(out2, ref) < 4e-3


def test_assemble_and_inject():
    ops = _ops()
    B, S, P, R, C = 2, 3, 16, 4, 128
    K, T = B * S, P + R + 1
    patch, cam, reg = randn(K, P, C, seed=1), randn(2, C, seed=2), randn(2, R, C, seed=3)
    inj0, ph = randn(K, C, seed=4), randn(C, seed=5)
    has = torch.tensor([1, 0, 0, 1, 1, 0], device="cuda", dtype=torch.int32)
    x = torch.empty(K, T, C, device="cuda")
    ops.assemble_tokens(x, patch, cam, reg, inj0, ph, has, K, S, T, R, C)
    slot = torch.tensor([0, 1, 1, 0, 1, 1], device="cuda")
    ref = torch.cat([(cam[slot] + inj0)[:, None], reg[slot], patch + (1 - has.float())[:, None, None] * ph], 1)
    assert torch.equal(x, ref)
    inj = randn(K, C, seed=6)
    slotbuf = torch.zeros(K * T, 2 * C, device="cuda", dtype=BF16)
    camout = torch.zeros(K, 2 * C, device="cuda")
    ops.inject_snapshot(x, inj, slotbuf, camout, K, T, C, C)
    ref[:, 0] += inj
    assert torch.equal(x, ref)
    assert torch.equal(slotbuf[:, C:], ref.reshape(K * T, C).to(BF16)) and (slotbuf[:, :C] == 0).all()
    assert torch.equal(camout[:, C:], ref[:, 0])
    # layers without a snapshot: only the camera-token rows are touched (one block per frame)
    inj2 = randn(K, C, seed=7)
    cam2 = torch.zeros(K, 2 * C, device="cuda")
    ops.inject_snapshot(x, inj2, None, cam2, K, T, C, 0)
    ref[:, 0] += inj2
    assert torch.equal(x, ref) and torch.equal(cam2[:, :C], ref[:, 0]) and (cam2[:, C:] == 0).all()


def test_depth_im2col_matches_reference_normalisation():
    ops = _ops()
    B, S, H, W, patch = 2, 4, 28, 42, 14
    idx = torch.tensor([0, 2, 3], device="cuda", dtype=torch.int32)
    depth = 0.5 + 4 * torch.rand(B, S, H, W, device="cuda")
    mask = (torch.rand(B, S, H, W, device="cuda") > 0.3).float()
    mask[1] = 0          # scene without valid pixels -> zeros (omnivggt_aggregator.py:121-122)
    Sd, hp, wp = 3, H // patch, W // patch
    cols = torch.zeros(B * Sd * hp * wp, 2 * patch * patch, device="cuda", dtype=BF16)
    scratch = torch.zeros(_ops().L.DEPTH_SCRATCH_DOUBLES(B), device="cuda", dtype=torch.float64)
    ops.depth_im2col(depth, mask, idx, scratch, cols, B, S, Sd, H, W, patch)
    d, m = depth[:, idx.long()], mask[:, idx.long()]
    norm = torch.zeros_like(d)
    for b in range(B):
        valid = d[b][m[b] > 0]
        if valid.numel():
            norm[b] = d[b] / (valid.mean() + 1e-8) * m[b]
    dm = torch.stack([norm.reshape(-1, H, W), m.reshape(-1, H, W)], 1)
    ref = F.unfold(dm, kernel_size=patch, stride=patch).transpose(1, 2).reshape(-1, 2 * patch * patch)
    assert rel(cols, ref) < 4e-3


# ----------------------------------------------------------------------------------------------- conv family
def _to_pad(x):  # NCHW fp32 -> zero-bordered NHWC bf16 [F,h+2,w+2,C]
    return F.pad(x.permute(0, 2, 3, 1), (0, 0, 1, 1, 1, 1)).to(BF16).contiguous()


def _from_pad(p):  # -> NCHW fp32 interior
    return p[:, 1:-1, 1:-1].float().permute(0, 3, 1, 2)


@pytest.mark.parametrize("Fr,h,w,Cin,Cout,bn", [(2, 9, 7, 64, 64, 0), (1, 37, 37, 256, 256, 0), (2, 19, 19, 128, 32, 0),
                                                (1, 37, 37, 256, 256, 512), (3, 20, 31, 128, 256, 512), (2, 30, 30, 256, 128, 384)])
def test_conv3x3_taps_with_skips_relu(Fr, h, w, Cin, Cout, bn):
    """3x3 conv as 9 row-shifted GEMMs over the zero-bordered layout + bias + two skips + ReLU
    (heads/dpt_head.py:379-399)."""
    ops = _ops()
    x = randn(Fr, Cin, h, w, seed=1)
    wt = randn(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    bias = randn(Cout, seed=3)
    s1, s2 = randn(Fr, Cout, h, w, seed=4), randn(Fr, Cout, h, w, seed=5)
    xp, s1p, s2p = _to_pad(x), _to_pad(s1), _to_pad(s2)
    wb = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).to(BF16).contiguous()
    outp = torch.full((Fr, h + 2, w + 2, Cout), 7.0, device="cuda", dtype=BF16)
    taps = [(ky - 1) * (w + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    ops.gemm(xp.reshape(-1, Cin), wb, taps=taps, epi=ops.L.EPI_BF16, bias=bias, act=ops.L.ACT_RELU, out=outp,
             ldo=Cout, skip1=s1p, skip2=s2p, rowmap=ops.L.ROWS_PAD, gh=h, gw=w, block_n=bn)
    ref = F.relu(F.conv2d(xp[:, 1:-1, 1:-1].float().permute(0, 3, 1, 2), wb.float().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2),
                          bias, padding=1) + s1p[:, 1:-1, 1:-1].float().permute(0, 3, 1, 2) + s2p[:, 1:-1, 1:-1].float().permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    assert rel(_from_pad(outp), ref) < 6e-3
    border = outp.clone()
    border[:, 1:-1, 1:-1] = 0
    assert (border == 0).all()         # border rows are rewritten as zeros


@pytest.mark.parametrize("ps,Cin,Cout,h,w,bn", [(4, 64, 64, 5, 3, 0), (2, 128, 128, 4, 4, 0), (4, 256, 256, 37, 37, 0),
                                                (4, 256, 256, 37, 37, 512)])
def test_conv_transpose_pixel_shuffle(ps, Cin, Cout, h, w, bn):
    """ConvTranspose2d(k = s) as one GEMM with a pixel-shuffle store (heads/dpt_head.py:84-89)."""
    ops = _ops()
    Fr = 2
    x = randn(Fr, Cin, h, w, seed=1)
    wt = randn(Cin, Cout, ps, ps, scale=Cin ** -0.5, seed=2)
    bias = randn(Cout, seed=3)
    a = x.permute(0, 2, 3, 1).reshape(-1, Cin).to(BF16).contiguous()
    wb = wt.permute(2, 3, 1, 0).reshape(ps * ps * Cout, Cin).to(BF16).contiguous()
    outp = torch.zeros(Fr, h * ps + 2, w * ps + 2, Cout, device="cuda", dtype=BF16)
    ops.gemm(a, wb, epi=ops.L.EPI_BF16, bias=bias, out=outp, ldo=Cout, rowmap=ops.L.ROWS_PIXSHUF, gh=h, gw=w, ps=ps, cout=Cout, block_n=bn)
    ref = F.conv_transpose2d(a.float().reshape(Fr, h, w, Cin).permute(0, 3, 1, 2), wb.float().reshape(ps, ps, Cout, Cin).permute(3, 2, 0, 1),
                             bias, stride=ps)
    torch.cuda.synchronize()
    assert rel(_from_pad(outp), ref) < 6e-3


def test_dense2pad_with_table():
    ops = _ops()
    Fr, h, w, Cin, Cout = 3, 5, 7, 256, 128
    a = randn(Fr * h * w, Cin, seed=1, dtype=BF16)
    wb = randn(Cout, Cin, scale=Cin ** -0.5, seed=2, dtype=BF16)
    bias, table = randn(Cout, seed=3), randn(h * w, Cout, seed=4)
    outp = torch.zeros(Fr, h + 2, w + 2, Cout, device="cuda", dtype=BF16)
    ops.gemm(a, wb, epi=ops.L.EPI_BF16, bias=bias, table=table, table_rows=h * w, out=outp, ldo=Cout,
             rowmap=ops.L.ROWS_DENSE2PAD, gh=h, gw=w)
    ref = (a.float() @ wb.float().t() + bias).reshape(Fr, h * w, Cout) + table
    assert rel(outp[:, 1:-1, 1:-1].reshape(Fr, h * w, Cout), ref) < 6e-3


def test_im2col_s2_and_conv():
    ops = _ops()
    Fr, h, w, C, Cout = 2, 7, 5, 64, 64
    x = randn(Fr, C, h, w, seed=1)
    wt = randn(Cout, C, 3, 3, scale=(9 * C) ** -0.5, seed=2)
    src = x.permute(0, 2, 3, 1).to(BF16).contiguous()
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    cols = torch.empty(Fr * oh * ow, 9 * C, device="cuda", dtype=BF16)
    ops.im2col3x3s2(src, cols, Fr, h, w, C)
    wb = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * C).to(BF16).contiguous()
    out = ops.linear_bf16(cols, wb)
    ref = F.conv2d(src.float().permute(0, 3, 1, 2), wb.float().reshape(Cout, 3, 3, C).permute(0, 3, 1, 2), None, stride=2, padding=1)
    assert rel(out.float().reshape(Fr, oh, ow, Cout).permute(0, 3, 1, 2), ref) < 6e-3


@pytest.mark.parametrize("h,w,H,W,C", [(4, 4, 8, 8, 64), (19, 19, 37, 37, 256), (8, 12, 14, 21, 128), (1, 1, 3, 3, 64)])
def test_upsample_bilinear(h, w, H, W, C):
    ops = _ops()
    Fr = 2
    x = randn(Fr, C, h, w, seed=1)
    tx, ty = randn(W, C // 2, seed=2), randn(H, C // 2, seed=3)
    xp = _to_pad(x)
    dst = torch.full((Fr, H + 2, W + 2, C), 3.0, device="cuda", dtype=BF16)
    ops.upsample_bilinear(xp, dst, tx, ty, Fr, h, w, H, W, C)
    ref = F.interpolate(xp[:, 1:-1, 1:-1].float().permute(0, 3, 1, 2), size=(H, W), mode="bilinear", align_corners=True)
    table = torch.cat([tx[None, :, :].expand(H, W, C // 2), ty[:, None, :].expand(H, W, C // 2)], -1)
    ref = ref + table.permute(2, 0, 1)
    assert rel(_from_pad(dst), ref) < 5e-3
    b = dst.clone()
    b[:, 1:-1, 1:-1] = 0
    assert (b == 0).all()


@pytest.mark.parametrize("outc,act", [(2, 0), (4, 1)])
def test_head_tail(outc, act):
    """3x3 conv 128->32 + ReLU + 1x1 32->outc + activations (heads/dpt_head.py:121-126; heads/head_act.py:61-125)."""
    ops = _ops()
    Fr, h, w, Cin = 2, 14, 28, 128
    x = randn(Fr, Cin, h, w, seed=1)
    w1 = randn(32, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    b1 = randn(32, scale=0.1, seed=3)
    w2 = randn(outc, 32, scale=32 ** -0.5, seed=4)
    b2 = randn(outc, scale=0.1, seed=5)
    xp = _to_pad(x)
    wb = w1.permute(0, 2, 3, 1).reshape(32, 9 * Cin).to(BF16).contiguous()
    preds = torch.zeros(Fr, h, w, outc - 1, device="cuda")
    conf = torch.zeros(Fr, h, w, device="cuda")
    taps = [(ky - 1) * (w + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    ops.gemm(xp.reshape(-1, Cin), wb, taps=taps, epi=ops.L.EPI_HEADTAIL, bias=b1, w2=w2.contiguous(), b2=b2, outc=outc,
             head_act=act, preds=preds, conf=conf, rowmap=ops.L.ROWS_PAD, gh=h, gw=w)
    y = F.conv2d(xp[:, 1:-1, 1:-1].float().permute(0, 3, 1, 2), wb.float().reshape(32, 3, 3, Cin).permute(0, 3, 1, 2), b1, padding=1)
    y = F.conv2d(F.relu(y), w2[:, :, None, None], b2).permute(0, 2, 3, 1)
    pr = torch.exp(y[..., :-1]) if act == 0 else torch.sign(y[..., :-1]) * torch.expm1(y[..., :-1].abs())
    torch.cuda.synchronize()
    assert rel(preds, pr) < 1e-2 and rel(conf, 1 + y[..., -1].exp()) < 1e-2


# ----------------------------------------------------------------------------------------------- fp16 mode of the DPT kernels
# The DPT heads run with IEEE-half operands / maps by default (ovg_gemm_args.f16, ovg_dpt_desc.f16): same kernels, the instruction
# descriptor's operand format and the 16-bit pack / unpack differ.  fp16 rounds to 2^-12 relative: tolerances are 8 x tighter.
F16 = torch.float16


@pytest.mark.parametrize("M,N,K,bn", [(300, 256, 128, 0), (1000, 384, 192, 128), (77, 96, 392, 64), (2748, 1024, 1024, 512),
                                      (5000, 1024, 128, 512), (2748, 384, 192, 384)])
def test_fp16_gemm_bias_gelu(M, N, K, bn):
    ops = _ops()
    a = randn(M, K, seed=1, dtype=F16)
    w = randn(N, K, scale=K ** -0.5, seed=2, dtype=F16)
    bias = randn(N, seed=3)
    out = torch.empty(M, N, device="cuda", dtype=F16)
    ops.gemm(a, w, epi=ops.L.EPI_BF16, bias=bias, act=ops.L.ACT_GELU, out=out, ldo=N, block_n=bn)
    ref = F.gelu(a.float() @ w.float().t() + bias)
    torch.cuda.synchronize()
    assert rel(out, ref) < 8e-4


@pytest.mark.parametrize("Fr,h,w,Cin,Cout,bn", [(2, 9, 7, 64, 64, 0), (1, 37, 37, 256, 256, 512), (2, 30, 30, 256, 128, 384)])
def test_fp16_conv3x3_taps_with_skips_relu(Fr, h, w, Cin, Cout, bn):
    ops = _ops()
    x = randn(Fr, Cin, h, w, seed=1)
    wt = randn(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    bias = randn(Cout, seed=3)
    s1, s2 = randn(Fr, Cout, h, w, seed=4), randn(Fr, Cout, h, w, seed=5)
    xp, s1p, s2p = _to_pad(x).to(F16), _to_pad(s1).to(F16), _to_pad(s2).to(F16)
    wb = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).to(F16).contiguous()
    outp = torch.full((Fr, h + 2, w + 2, Cout), 7.0, device="cuda", dtype=F16)
    taps = [(ky - 1) * (w + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    ops.gemm(xp.reshape(-1, Cin), wb, taps=taps, epi=ops.L.EPI_BF16, bias=bias, act=ops.L.ACT_RELU, out=outp,
             ldo=Cout, skip1=s1p, skip2=s2p, rowmap=ops.L.ROWS_PAD, gh=h, gw=w, block_n=bn)
    ref = F.relu(F.conv2d(_from_pad(xp), wb.float().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2), bias, padding=1)
                 + _from_pad(s1p) + _from_pad(s2p))
    torch.cuda.synchronize()
    assert rel(_from_pad(outp), ref) < 8e-4
    border = outp.clone()
    border[:, 1:-1, 1:-1] = 0
    assert (border == 0).all()


def test_fp16_stores_saturate_instead_of_overflowing():
    """|acc| > 65504 is stored as +-65504, never inf (cvt.rn.satfinite.f16x2.f32)."""
    ops = _ops()
    a = torch.full((256, 64), 64.0, device="cuda", dtype=F16)
    w = torch.full((64, 64), 32.0, device="cuda", dtype=F16)
    w[1::2] = -32.0
    out = torch.empty(256, 64, device="cuda", dtype=F16)
    ops.gemm(a, w, epi=ops.L.EPI_BF16, out=out, ldo=64)          # acc = +-131072
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert (out[:, 0::2] == 65504).all() and (out[:, 1::2] == -65504).all()


@pytest.mark.parametrize("h,w,H,W,C", [(4, 4, 8, 8, 64), (19, 19, 37, 37, 256), (8, 12, 14, 21, 144)])
def test_fp16_upsample_bilinear(h, w, H, W, C):
    ops = _ops()
    Fr = 2
    x = randn(Fr, C, h, w, seed=1)
    tx, ty = randn(W, C // 2, seed=2), randn(H, C // 2, seed=3)
    xp = _to_pad(x).to(F16)
    dst = torch.full((Fr, H + 2, W + 2, C), 3.0, device="cuda", dtype=F16)
    ops.upsample_bilinear(xp, dst, tx, ty, Fr, h, w, H, W, C)
    ref = F.interpolate(_from_pad(xp), size=(H, W), mode="bilinear", align_corners=True)
    table = torch.cat([tx[None, :, :].expand(H, W, C // 2), ty[:, None, :].expand(H, W, C // 2)], -1)
    assert rel(_from_pad(dst), ref + table.permute(2, 0, 1)) < 6e-4
    b = dst.clone()
    b[:, 1:-1, 1:-1] = 0
    assert (b == 0).all()


def test_fp16_layernorm_out_and_head_tail():
    ops = _ops()
    C, T, P = 2048, 21, 16
    xb = randn(4 * T, C, seed=4, dtype=BF16)
    out = torch.empty(4 * P, C, device="cuda", dtype=F16)
    ops.layernorm(xb, out, None, None, 1e-5, grp_out=P, grp_in=T, grp_off=5)
    ref = F.layer_norm(xb.float().reshape(4, T, C)[:, 5:], (C,), None, None, 1e-5).reshape(4 * P, C)
    assert rel(out, ref) < 5e-4
    Fr, h, w, Cin, outc = 2, 14, 28, 128, 4
    x = randn(Fr, Cin, h, w, seed=1)
    w1 = randn(32, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    b1, w2, b2 = randn(32, scale=0.1, seed=3), randn(outc, 32, scale=32 ** -0.5, seed=4), randn(outc, scale=0.1, seed=5)
    xp = _to_pad(x).to(F16)
    wb = w1.permute(0, 2, 3, 1).reshape(32, 9 * Cin).to(F16).contiguous()
    preds = torch.zeros(Fr, h, w, outc - 1, device="cuda")
    conf = torch.zeros(Fr, h, w, device="cuda")
    taps = [(ky - 1) * (w + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    ops.gemm(xp.reshape(-1, Cin), wb, taps=taps, epi=ops.L.EPI_HEADTAIL, bias=b1, w2=w2.contiguous(), b2=b2, outc=outc,
             head_act=1, preds=preds, conf=conf, rowmap=ops.L.ROWS_PAD, gh=h, gw=w)
    y = F.conv2d(_from_pad(xp), wb.float().reshape(32, 3, 3, Cin).permute(0, 3, 1, 2), b1, padding=1)
    y = F.conv2d(F.relu(y), w2[:, :, None, None], b2).permute(0, 2, 3, 1)
    pr = torch.sign(y[..., :-1]) * torch.expm1(y[..., :-1].abs())
    torch.cuda.synchronize()
    assert rel(preds, pr) < 1e-4 and rel(conf, 1 + y[..., -1].exp()) < 1e-4


@pytest.mark.parametrize("dtype", [F16, BF16])
@pytest.mark.parametrize("Fr,h,w,H,W,outc,act", [(2, 12, 20, 21, 35, 2, 0), (2, 80, 90, 140, 300, 4, 1), (3, 9, 75, 16, 131, 4, 1),
                                               (1, 296, 296, 518, 518, 2, 0), (2, 37, 37, 37, 64, 4, 1)])
def test_dpt_tail_fused(Fr, h, w, H, W, outc, act, dtype):
    """ovg_dpt_tail: resize + position embedding + 3x3 conv 128->32 + ReLU + 1x1 + activations in one kernel (the H x W x 128 map
    is never written) against PyTorch fp32 (heads/dpt_head.py:242-260), and against the two-kernel path it replaces."""
    ops = _ops()
    Cin = 128
    assert ops.L.lib().ovg_dpt_tail_supported(h, w, H, W, Cin) == 1
    x = randn(Fr, Cin, h, w, seed=1)
    w1 = randn(32, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    b1, w2, b2 = randn(32, scale=0.1, seed=3), randn(outc, 32, scale=32 ** -0.5, seed=4), randn(outc, scale=0.1, seed=5)
    tx, ty = randn(W, Cin // 2, scale=0.1, seed=6), randn(H, Cin // 2, scale=0.1, seed=7)
    xp = _to_pad(x).to(dtype)
    wb = w1.permute(0, 2, 3, 1).reshape(32, 9 * Cin).to(dtype).contiguous()
    preds, conf = ops.dpt_tail(xp, tx, ty, wb, b1, w2.contiguous(), b2, act, Fr, h, w, H, W)
    torch.cuda.synchronize()
    up = F.interpolate(_from_pad(xp), size=(H, W), mode="bilinear", align_corners=True)
    up = up.to(dtype).float()                          # the kernel rounds the resized operand to 16 bits; the embedding stays fp32
    up = up + torch.cat([tx[None, :, :].expand(H, W, Cin // 2), ty[:, None, :].expand(H, W, Cin // 2)], -1).permute(2, 0, 1)
    y = F.conv2d(up, wb.float().reshape(32, 3, 3, Cin).permute(0, 3, 1, 2), b1, padding=1)
    y = F.conv2d(F.relu(y), w2[:, :, None, None], b2).permute(0, 2, 3, 1)
    pr = torch.exp(y[..., :-1]) if act == 0 else torch.sign(y[..., :-1]) * torch.expm1(y[..., :-1].abs())
    tol = 2e-3 if dtype == F16 else 1.2e-2              # re-rounding of `up` may differ by one ulp of the 16-bit type from torch's
    assert torch.isfinite(preds).all() and torch.isfinite(conf).all()
    assert rel(preds, pr) < tol and rel(conf, 1 + y[..., -1].exp()) < tol, (rel(preds, pr), rel(conf, 1 + y[..., -1].exp()))
    # the path it replaces: ovg_upsample_bilinear -> HEADTAIL GEMM
    dst = torch.zeros(Fr, H + 2, W + 2, Cin, device="cuda", dtype=dtype)
    ops.upsample_bilinear(xp, dst, tx, ty, Fr, h, w, H, W, Cin)
    p2 = torch.zeros(Fr, H, W, outc - 1, device="cuda")
    c2 = torch.zeros(Fr, H, W, device="cuda")
    taps = [(ky - 1) * (W + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    ops.gemm(dst.reshape(-1, Cin), wb, taps=taps, epi=ops.L.EPI_HEADTAIL, bias=b1, w2=w2.contiguous(), b2=b2, outc=outc,
             head_act=act, preds=p2, conf=c2, rowmap=ops.L.ROWS_PAD, gh=H, gw=W)
    torch.cuda.synchronize()
    tol2 = 1e-3 if dtype == F16 else 8e-3              # that path rounds (map + embedding) to 16 bits, this one the map only
    assert rel(preds, p2) < tol2 and rel(conf, c2) < tol2, (rel(preds, p2), rel(conf, c2))


# ----------------------------------------------------------------------------------------------- C host
def test_c_host_drives_the_runtime(tmp_path):
    """A plain C program (tests/c/runtime_identity.c: gcc, libovg + libcudart, no Python / torch in the process) runs the
    aggregator through the handle-level C ABI with raw device pointers; with zero block weights the kept intermediates must
    equal the assembled tokens bit for bit."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "omnivggt-official_b200")
    exe = str(tmp_path / "runtime_identity")
    cuda_lib = "/usr/local/cuda/lib64"
    subprocess.check_call(["gcc", os.path.join(root, "tests", "c", "runtime_identity.c"), "-I", os.path.join(root, "include"),
                           "-L", pkg, "-lovg", "-L", cuda_lib, "-lcudart", "-lm", f"-Wl,-rpath,{pkg}", f"-Wl,-rpath,{cuda_lib}",
                           "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 mismatches" in r.stdout


# ----------------------------------------------------------------------------------------------- context-parallel pieces (one GPU)
def test_attention_own_queries_against_all_keys():
    """ovg_attention with nq < nkv: a window of the query rows against ALL keys equals the same rows of the full self-attention bit
    for bit (what a rank of the context-parallel global block computes)."""
    ops = _ops()
    heads, n, lo, hi = 4, 1374 * 2, 1374, 1374 + 700
    q = randn(1, heads, n, 64, seed=1, dtype=BF16) * 0.18
    k = randn(1, heads, n, 64, seed=2, dtype=BF16)
    v = randn(1, heads, n, 64, seed=3, dtype=BF16)
    full = torch.zeros(1, n, heads * 64, device="cuda", dtype=BF16)
    ops.attention(q, k, v, full, 1, heads, n)
    part = torch.zeros(1, hi - lo, heads * 64, device="cuda", dtype=BF16)
    ops.attention(q[:, :, lo:hi].contiguous(), k, v, part, 1, heads, hi - lo, n)
    torch.cuda.synchronize()
    assert torch.equal(part, full[:, lo:hi])
    # the shape a rank of a 2-GPU context-parallel forward runs (half of the query rows of 8 views against all keys): 688 tiles,
    # the 96 of the last wave split over the keys
    heads, n = 16, 8 * 1374
    q = randn(1, heads, n // 2, 64, seed=4, dtype=BF16) * 0.18
    k = randn(1, heads, n, 64, seed=5, dtype=BF16)
    v = randn(1, heads, n, 64, seed=6, dtype=BF16)
    plain = torch.zeros(1, n // 2, heads * 64, device="cuda", dtype=BF16)
    split = torch.zeros_like(plain)
    ops.attention(q, k, v, plain, 1, heads, n // 2, n)
    ops.attention(q, k, v, split, 1, heads, n // 2, n, scratch=ops.attention_scratch("cuda"))
    torch.cuda.synchronize()
    assert not torch.equal(plain, split) and rel(split, plain) < 4e-3


def test_qkv_epilogue_stores_kv_rows_into_peer_buffers():
    """EPI_QKV with k_peers / v_peers: the K / V rows of this rank's tokens land in every listed full-length buffer at the rank's
    token offset (here both "peers" are local allocations) and equal what the plain epilogue writes; q stays local."""
    ops = _ops()
    C, T, frames, hp, wp = 256, 25, 2, 4, 5
    heads, M = C // 64, frames * T
    a = randn(M, C, seed=1, dtype=BF16)
    w = randn(3 * C, C, scale=C ** -0.5, seed=2, dtype=BF16)
    bias = randn(3 * C, scale=0.1, seed=3)
    ln = [1 + 0.1 * randn(64, seed=4), 0.1 * randn(64, seed=5), 1 + 0.1 * randn(64, seed=6), 0.1 * randn(64, seed=7)]
    cos, sin = ops.rope_tables(max(hp, wp) + 1, "cuda")
    q0, k0, v0 = (torch.zeros(1, heads, M, 64, device="cuda", dtype=BF16) for _ in range(3))
    ops.qkv_proj(a, w, bias, *ln, q0, k0, v0, ntok=M, T=T, nspecial=5, wp=wp, rope_cos=cos, rope_sin=sin)
    total, off = 3 * M, M                       # this "rank" owns tokens [M, 2M) of a 3M-token scene
    peers_k = [torch.full((1, heads, total, 64), 7.0, device="cuda", dtype=BF16) for _ in range(2)]
    peers_v = [torch.full((1, heads, total, 64), 7.0, device="cuda", dtype=BF16) for _ in range(2)]
    q1 = torch.zeros_like(q0)
    import ctypes
    kp = (ctypes.c_void_p * 8)(*[t.data_ptr() for t in peers_k])
    vp = (ctypes.c_void_p * 8)(*[t.data_ptr() for t in peers_v])
    ops.gemm(a, w, epi=ops.L.EPI_QKV, bias=bias, q_out=q1, k_out=None, v_out=None, C=C, ntok=M, T=T, nspecial=5, wp=wp,
             maxpos=cos.shape[0], qn_w=ln[0], qn_b=ln[1], kn_w=ln[2], kn_b=ln[3], rope_cos=cos, rope_sin=sin, qk_norm=1, rope=1,
             qscale=(1.0 / math.sqrt(64.0)) * math.log2(math.e), k_peers=kp, v_peers=vp, n_peers=2, peer_ntok=total, peer_tok_off=off)
    torch.cuda.synchronize()
    assert torch.equal(q1, q0)
    for pk, pv in zip(peers_k, peers_v):
        assert torch.equal(pk[:, :, off:off + M], k0) and torch.equal(pv[:, :, off:off + M], v0)
        assert (pk[:, :, :off] == 7.0).all() and (pk[:, :, off + M:] == 7.0).all() and (pv[:, :, :off] == 7.0).all()


def test_peer_barrier_single_rank_and_epoch():
    """The flag barrier with world = 1 must pass immediately and bump the device epoch once per call (graph-replay safe)."""
    from omnivggt_official_b200 import _lib as L
    import ctypes
    flags = torch.zeros(8, dtype=torch.int32, device="cuda")
    epoch = torch.zeros(1, dtype=torch.int32, device="cuda")
    fp = (ctypes.c_void_p * 8)(flags.data_ptr())
    for _ in range(3):
        L.check(L.lib().ovg_peer_barrier(fp, epoch.data_ptr(), 0, 1, L.stream()))
    torch.cuda.synchronize()
    assert int(epoch.item()) == 3 and int(flags[0].item()) == 3
