"""fp64 references of the hot-path kernels, with per-element error bounds taken from where each kernel rounds.

Covers the GEMM and its epilogues, the QKV epilogue, attention, LayerNorm, the camera head, and the kernels of the DPT output:
bilinear upsampling, the fused output tail, and the im2col copies of the patch embeddings.  Only the maths is restated here
(pure torch, float64 unless stated).  tests/test_kernel_bounds_gpu.py and tests/test_dpt_bounds_gpu.py check the CUDA kernels
against these functions, and tests/test_kernel_ref_cpu.py and tests/test_dpt_ref_cpu.py check the functions themselves: CPU
emulations of each kernel's arithmetic must pass, and emulations with seeded mistakes must fail.

Where the bounds come from:
  * A 16-bit store is allowed one unit in the last place (ulp) of the stored type at the reference's magnitude.  That is a full ulp,
    not half: a value rounded once in fp32 and again to 16 bits can land one ulp away.
  * fp32 tensor-core accumulation over K terms is allowed ACC_C * sqrt(K) * 2^-24 * sum_k |a_k||b_k|.  The tensor cores' fp32
    accumulation need not round like IEEE fp32, so ACC_C is not derived: it is measured (see ACC_C).
  * Attention rounds the probabilities P to bf16 for the P.V MMA, but sums the row sum l from the unrounded fp32 values.  An output
    element can therefore move by U_BF16 * sum_j p_j |v_jd| / l, where U_BF16 = 2^-8 is bf16's unit roundoff (8 significant bits).
    The P.V accumulation, the store, the score error (a score error ds scales p by 2^ds) and ex2.approx come on top.
The helpers return the worst ratio of error to bound and where it occurs, so a failing test names the row, column or head.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import torch

F64 = torch.float64
F32 = torch.float32
U_BF16 = 2.0 ** -8          # unit roundoff of bf16 (8 significant bits)
EPS32 = 2.0 ** -24          # unit roundoff of fp32

# Accumulation constant of the wgmma fp32 accumulators.  test_gemm_accumulation_constant measures the largest
# |acc - exact| / (sqrt(K) 2^-24 sum|a||b|) over random bf16 GEMMs with K = 64 .. 4096: 0.248 on an H100 80GB HBM3 (132 SMs,
# 700 W), at K = 64; 0.16 - 0.21 at K = 192 .. 4096.  ACC_C = 2 keeps a factor of 8 above that, and the test requires 4.
ACC_C = 2.0

_BITS = {torch.bfloat16: (8, -126), torch.float16: (11, -14), torch.float32: (24, -126)}   # significant bits, min normal exponent


def ulp(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """One ulp of `dtype` at |x| (fp64); below the normal range, the subnormal spacing."""
    bits, emin = _BITS[dtype]
    x = x.to(F64)
    _, e = torch.frexp(x)                       # |x| = m 2^e with 0.5 <= m < 1, so floor(log2 |x|) = e - 1
    e = torch.where(x == 0, float(emin), torch.clamp(e.to(F64) - 1, min=emin))
    return torch.exp2(e - (bits - 1))


def round_to(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """fp64 -> `dtype` with round-to-nearest-even (fp16 saturating at +-65504, as cvt.rn.satfinite), back to fp64.  Exact for
    inputs that fp32 holds exactly; others may be rounded twice."""
    x = x.to(F64)
    if dtype == torch.float16:
        x = x.clamp(-65504.0, 65504.0)
    return x.to(dtype).to(F64)


def is_tie(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """x lies exactly halfway between two neighbouring values of `dtype` (x itself is not one)."""
    x = x.to(F64)
    u = ulp(x, dtype)
    return (torch.remainder(x, u) == u / 2) & (round_to(x, dtype) != x)


# ----------------------------------------------------------------------------------------------- checks
def worst(err: torch.Tensor, bound: torch.Tensor) -> Tuple[float, Tuple[int, ...]]:
    """(max of err / bound, index of that element).  A zero bound demands a zero error."""
    err, bound = err.to(F64), bound.to(F64)
    r = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, torch.inf, 0.0))
    r = torch.nan_to_num(r, nan=torch.inf)
    i = int(torch.argmax(r.reshape(-1)))
    return float(r.reshape(-1)[i]), tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape))


def bound_ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> Tuple[float, Tuple[int, ...]]:
    """Worst |out - ref| / bound (a non-finite output counts as infinitely far)."""
    o = out.to(F64).cpu()
    err = torch.where(torch.isfinite(o), (o - ref.cpu()).abs(), torch.full_like(o, torch.inf))
    return worst(err, bound.cpu())


def match_fraction(out: torch.Tensor, ref: torch.Tensor, dtype: torch.dtype) -> float:
    """Fraction of the 16-bit outputs that equal the fp64 reference rounded once to `dtype`."""
    return float((out.to(F64).cpu() == round_to(ref.cpu(), dtype)).double().mean())


def check_bound(out, ref, bound, what: str, dims: Sequence[str] = ()) -> float:
    """Assert |out - ref| <= bound element-wise; returns the worst ratio (the margin a PR reports)."""
    r, at = bound_ratio(out, ref, bound)
    where = ", ".join(f"{d}={i}" for d, i in zip(dims, at)) if dims else str(at)
    assert r <= 1.0, f"{what}: error {r:.3g} x its bound at {where} (out {float(out.reshape(-1)[_flat(at, out.shape)]):.9g}, " \
                     f"ref {float(ref.reshape(-1)[_flat(at, ref.shape)]):.9g})"
    return r


def check_rounded(out, ref, bound, dtype, what: str, dims: Sequence[str] = (), min_match: float = 0.99) -> Tuple[float, float]:
    """16-bit output: within the bound everywhere, and at least `min_match` of the elements equal round(ref) (round-to-nearest-even
    gives nearly all; truncation gives about half, which a bound of one ulp cannot see)."""
    r = check_bound(out, ref, bound, what, dims)
    f = match_fraction(out, ref, dtype)
    assert f >= min_match, f"{what}: only {f:.4f} of the outputs equal the fp64 reference rounded to {dtype}"
    return r, f


def _flat(at, shape) -> int:
    i = 0
    for a, s in zip(at, shape):
        i = i * s + a
    return i


# ----------------------------------------------------------------------------------------------- GEMM
def gemm_acc(a: torch.Tensor, b: torch.Tensor, taps: Sequence[int] = (0,), m: Optional[int] = None):
    """acc[r, n] = sum_t A[r + taps[t]] . B[n, t K:(t+1) K] with A rows outside [0, rows) read as zero (the TMA fill), and the
    matching sum of |a||b|.  Returns (acc, absacc), fp64 [m, N]."""
    a, b = a.to(F64), b.to(F64)
    rows, K = a.shape
    m = rows if m is None else m
    acc = torch.zeros(m, b.shape[0], dtype=F64, device=a.device)
    absacc = torch.zeros_like(acc)
    r = torch.arange(m, device=a.device)
    for t, off in enumerate(taps):
        src = r + off
        ok = (src >= 0) & (src < rows)
        at = torch.zeros(m, K, dtype=F64, device=a.device)
        at[ok] = a[src[ok]]
        bt = b[:, t * K:(t + 1) * K]
        acc += at @ bt.t()
        absacc += at.abs() @ bt.abs().t()
    return acc, absacc


def int_operands(rows: int, n: int, K: int, seed: int, lim: int = 8, extra_cols: int = 0):
    """Small-integer GEMM operands (|a|, |b| <= lim, fp64 on the CPU): a [rows, K + extra_cols], b [n, K].  With K * lim^2 < 2^18
    every partial sum is an integer below 2^18 in any summation order, so fp32 accumulation is exact."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(-lim, lim + 1, (rows, K + extra_cols), generator=g).to(F64)
    b = torch.randint(-lim, lim + 1, (n, K), generator=g).to(F64)
    return a, b


def acc_bound(absacc: torch.Tensor, K: int) -> torch.Tensor:
    """What fp32 tensor-core accumulation over K terms may add to a dot product with sum |a||b| = absacc."""
    return ACC_C * math.sqrt(K) * EPS32 * absacc


def gelu(x: torch.Tensor) -> torch.Tensor:
    """Exact-erf GELU (nn.GELU())."""
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def gelu_bound(x: torch.Tensor, ex: torch.Tensor) -> torch.Tensor:
    """Error of the kernel's GELU at x when x itself is off by ex: |GELU'| <= 1.13, the erf approximation (Abramowitz-Stegun
    7.1.26, |error| <= 1.5e-7) scaled by |x| / 2, and ~8 fp32 roundings / MUFU approximations."""
    return 1.13 * ex + x.abs() * (0.5 * 1.5e-7 + 8 * EPS32)


def linear_ref(a, w, bias=None, act: str = "none", out_dtype=torch.bfloat16):
    """out = act(a w^T + bias) stored in `out_dtype`: (ref fp64, per-element bound)."""
    acc, absacc = gemm_acc(a, w)
    x = acc + (bias.to(F64)[None] if bias is not None else 0.0)
    ex = acc_bound(absacc, a.shape[1]) + 2 * EPS32 * x.abs()
    if act == "gelu":
        ref, e = gelu(x), gelu_bound(x, ex)
    elif act == "relu":
        ref, e = x.clamp(min=0), ex
    else:
        ref, e = x, ex
    return ref, e + ulp(ref, out_dtype)


def qkv_ref(a, w, bias, heads: int, ntok: int, qscale: float, ln: Optional[Sequence[torch.Tensor]] = None,
            rope: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None, eps: float = 1e-5):
    """EPI_QKV: (q, k, v) refs fp64 [nb, heads, ntok, 64] and their bounds.  ln = (qn_w, qn_b, kn_w, kn_b) for the q/k
    LayerNorm(64); rope = (cos, sin, pos) with fp32 tables [maxpos, 16] and integer positions pos [M, 2] (row, column)."""
    M, C = a.shape[0], w.shape[1]
    acc, absacc = gemm_acc(a, w)
    t = acc + bias.to(F64)[None]
    et = acc_bound(absacc, C) + EPS32 * t.abs()
    t = t.reshape(M, 3, heads, 64)
    et = et.reshape(M, 3, heads, 64)
    outs, bnds = [], []
    for which in range(3):
        x, ex = t[:, which], et[:, which]
        if which < 2 and ln is not None:
            wgt, bb = ln[2 * which].to(F64), ln[2 * which + 1].to(F64)
            mean = x.mean(-1, keepdim=True)
            d = x - mean
            var = (d * d).mean(-1, keepdim=True)
            rstd = 1.0 / torch.sqrt(var + eps)
            xh = d * rstd
            emax = ex.amax(-1, keepdim=True)
            e_mean = emax + 64 * EPS32 * x.abs().amax(-1, keepdim=True)
            rel_r = e_mean * rstd + 2.0 ** -21
            exh = rstd * (ex + e_mean + 2 * EPS32 * d.abs()) + xh.abs() * rel_r
            x = xh * wgt + bb
            ex = exh * wgt.abs() + 2 * EPS32 * x.abs()
        if which == 0:
            x, ex = x * qscale, ex * abs(qscale) + EPS32 * (x * qscale).abs()
        if which < 2 and rope is not None:
            cos, sin, pos = rope
            cos, sin = cos.to(F64), sin.to(F64)
            y = x.clone()
            ey = ex.clone()
            for half, axis in ((0, 0), (32, 1)):
                c = cos[pos[:, axis].long()][:, None, :]       # [M, 1, 16]
                s = sin[pos[:, axis].long()][:, None, :]
                lo, hi = x[..., half:half + 16], x[..., half + 16:half + 32]
                elo, ehi = ex[..., half:half + 16], ex[..., half + 16:half + 32]
                y[..., half:half + 16] = lo * c - hi * s
                y[..., half + 16:half + 32] = hi * c + lo * s
                e = c.abs() * elo + s.abs() * ehi + 2 * EPS32 * ((lo * c).abs() + (hi * s).abs())
                e2 = c.abs() * ehi + s.abs() * elo + 2 * EPS32 * ((hi * c).abs() + (lo * s).abs())
                ey[..., half:half + 16], ey[..., half + 16:half + 32] = e, e2
            x, ex = y, ey
        nb = M // ntok
        x = x.reshape(nb, ntok, heads, 64).permute(0, 2, 1, 3)
        ex = ex.reshape(nb, ntok, heads, 64).permute(0, 2, 1, 3)
        outs.append(x)
        bnds.append(ex + ulp(x, torch.bfloat16))
    return outs, bnds


def headtail_ref(a, w, taps, bias, w2, b2, head_act: int, F: int, gh: int, gw: int):
    """EPI_HEADTAIL over the zero-bordered grid: 3x3 conv (row-shifted taps) + bias + ReLU, 1x1 32 -> outc, then the activations.
    Returns (preds [F,gh,gw,outc-1], conf [F,gh,gw], bound of preds, bound of conf), all fp64."""
    acc, absacc = gemm_acc(a, w, taps)
    K = a.shape[1] * len(taps)
    h = acc + bias.to(F64)[None]
    eh = acc_bound(absacc, K) + EPS32 * h.abs()
    pw = gw + 2
    r = torch.arange(acc.shape[0], device=acc.device)
    fr, rem = r // ((gh + 2) * pw), r % ((gh + 2) * pw)
    yy, xx = rem // pw, rem % pw
    inner = (yy >= 1) & (yy <= gh) & (xx >= 1) & (xx <= gw)
    return head_post(h[inner].reshape(F, gh, gw, -1), eh[inner].reshape(F, gh, gw, -1), w2, b2, head_act)


def head_post(h, eh, w2, b2, head_act: int, epi_c: float = 34.0):
    """ReLU -> 1x1 conv 32 -> outc -> activations (exp / inverse-log; confidence 1 + exp), from the 3x3 conv output h [..., 32]
    (fp64, bias included) and its error bound eh.  epi_c: fp32 roundings allowed to the 1x1 (0 when it is exact).  The
    activations may add 2 fp32 ulp (expf; expm1f 1 ulp).  Returns (preds [..., outc-1], conf [...], bound of preds, bound of conf)."""
    eh = torch.where(h > 0, eh, torch.where(h + eh > 0, eh, torch.zeros_like(eh)))
    h = h.clamp(min=0)
    w2, b2 = w2.to(device=h.device, dtype=F64), b2.to(device=h.device, dtype=F64)
    y = h @ w2.t() + b2
    ey = eh @ w2.abs().t() + epi_c * EPS32 * (h @ w2.abs().t() + b2.abs())
    yp, ep = y[..., :-1], ey[..., :-1]
    if head_act == 0:
        preds = torch.exp(yp)
        bp = preds * (torch.expm1(ep) + 4 * EPS32)
    else:
        preds = torch.sign(yp) * torch.expm1(yp.abs())
        bp = torch.exp(yp.abs()) * torch.expm1(ep) + torch.exp(yp.abs()) * ep + 4 * EPS32 * preds.abs()
    yc, ec = y[..., -1], ey[..., -1]
    conf = 1.0 + torch.exp(yc)
    bc = torch.exp(yc) * (torch.expm1(ec) + 4 * EPS32) + EPS32 * conf
    return preds, conf, bp, bc


# ----------------------------------------------------------------------------------------------- attention
def attention_ref(q, k, v):
    """softmax_j(q . k_j) v_j with q in log2 units (pre-scaled by log2(e)/sqrt(64)); q [B,H,nq,64], k, v [B,H,nkv,64].
    Returns (out fp64 [B, nq, H*64], bound fp64 [B, nq, H*64])."""
    q, k, v = q.to(F64), k.to(F64), v.to(F64)
    B, H, nq, D = q.shape
    nkv = k.shape[2]
    s = q @ k.transpose(-1, -2)
    m = s.amax(-1, keepdim=True)
    p = torch.exp2(s - m)
    l = p.sum(-1, keepdim=True)
    out = (p @ v) / l
    pv = (p @ v.abs()) / l                                     # sum_j p_j |v_jd| / l
    # score error: fp32 tensor-core accumulation of q . k over 64 terms, for the score and for the maximum it is measured from
    ds = 2 * ACC_C * 8.0 * EPS32 * (q.abs() @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True)
    ntiles = (nkv + 127) // 128
    rel_p = U_BF16 + math.log(2.0) * ds + 2.0 ** -21 + ACC_C * math.sqrt(nkv) * EPS32
    rel_l = (nkv / 4 + 2 * ntiles + 16) * EPS32 + math.log(2.0) * ds
    bound = pv * rel_p + out.abs() * rel_l
    out = out.permute(0, 2, 1, 3).reshape(B, nq, H * D)
    bound = bound.permute(0, 2, 1, 3).reshape(B, nq, H * D)
    return out, bound + ulp(out, torch.bfloat16)


def attention_path(batch: int, heads: int, nq: int, nkv: int, sms: int, scratch: bool) -> Tuple[str, int]:
    """Which path ovg_attention takes on a device with `sms` SMs, restated from its launch rule: ("persistent" | "plain" |
    "split", KV parts).  Tests assert the choice through the launch count and the scratch bytes the split writes."""
    tiles = -(-nq // 128) * batch * heads
    kv_tiles = -(-nkv // 128)
    if tiles > sms and kv_tiles <= 16:
        return "persistent", 1
    tail = tiles % sms
    parts = 1
    if scratch and tiles > sms and tail > 0 and kv_tiles >= 24:
        best = 1.0
        for c in (2, 3, 4):
            cost = (-(-(tail * c) // sms)) / c + 0.04
            if cost < best - 0.1:
                best, parts = cost, c
    return ("split", parts) if parts > 1 else ("plain", 1)


def split_scratch_bytes(batch: int, heads: int, nq: int, sms: int, parts: int) -> int:
    """Bytes of the scratch a split launch writes: (un-normalised O fp32 [128, 64] + (m, l)) per part of each tail tile."""
    tail = (-(-nq // 128) * batch * heads) % sms
    return tail * parts * 128 * (64 * 4 + 8)


def onehot_codes(n: int, generator: torch.Generator) -> torch.Tensor:
    """n distinct +-1 codes of 64 dimensions (fp64 [n, 64]).  Two distinct codes agree in at most 63 places, so with a query of
    128 x its target's code the target scores 128 * 64 and every other key at most 128 * 62: a gap of 256 in log2 units, which
    ex2 turns into an exact 0."""
    bits = torch.randint(0, 2, (n, 64), generator=generator, dtype=torch.int64)
    # force distinctness: the first 20 bits carry the index (n < 2^20)
    idx = torch.arange(n, dtype=torch.int64)
    for b in range(20):
        bits[:, b] = (idx >> b) & 1
    return bits.to(F64) * 2 - 1


def onehot_case(B: int, H: int, nq: int, nkv: int, seed: int):
    """Each query puts all its weight on one key: k = distinct +-1 codes, q_i = 128 x the code of key t_i.  Returns (q, k, v bf16
    [B,H,n,64] on the CPU, expected bf16 [B, nq, H*64] = v[t_i] bit for bit).  This checks the indexing of every row, head, batch
    entry and ragged tile, and the rescale when the maximum arrives late (t_i anywhere in the sequence)."""
    g = torch.Generator().manual_seed(seed)
    codes = torch.stack([torch.stack([onehot_codes(nkv, g) for _ in range(H)]) for _ in range(B)])       # [B,H,nkv,64]
    tgt = torch.randint(0, nkv, (B, H, nq), generator=g)
    q = 128.0 * torch.gather(codes, 2, tgt[..., None].expand(-1, -1, -1, 64))
    v = torch.randn(B, H, nkv, 64, generator=g, dtype=F64).to(torch.bfloat16)
    exp = torch.gather(v, 2, tgt[..., None].expand(-1, -1, -1, 64)).permute(0, 2, 1, 3).reshape(B, nq, H * 64)
    return q.to(torch.bfloat16), codes.to(torch.bfloat16), v, exp


def uniform_case(B: int, H: int, n: int, seed: int):
    """Every score is exactly -16 (q = -16 e_0, k_j0 = 1), so every probability is exactly 1 and out = bf16(fp32(sum_j v_j) *
    fp32(1 / n)) on every path, with small-integer v summed exactly.  A key that the mask should drop scores 0 (it reads as zero)
    and takes nearly all the weight, so an off-by-one in the ragged tile cannot hide.  Returns (q, k, v, expected bf16)."""
    g = torch.Generator().manual_seed(seed)
    q = torch.zeros(B, H, n, 64, dtype=F64)
    q[..., 0] = -16.0
    k = torch.randint(-8, 9, (B, H, n, 64), generator=g).to(F64)
    k[..., 0] = 1.0
    v = torch.randint(-8, 9, (B, H, n, 64), generator=g).to(F64)
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(n), dtype=torch.float32)
    exp = (v.sum(2).float() * inv).to(torch.bfloat16)                                                 # [B, H, 64]
    exp = exp[:, :, None].expand(B, H, n, 64).permute(0, 2, 1, 3).reshape(B, n, H * 64)
    return q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16), exp


def rounding_case(B: int, H: int, n: int, seed: int):
    """Key 0 scores 0 and carries v; every other key scores -0.99609375 (p = 0.5013, which bf16 rounds to 0.5) and has v = 0.
    out = v_0 / l: exact when l sums the unrounded p, as the kernel does, but 0.27 % off when l sums the rounded ones, since all
    those roundings go the same way.  Returns (q, k, v bf16, reference fp64 [B, n, H*64])."""
    g = torch.Generator().manual_seed(seed)
    q = torch.zeros(B, H, n, 64, dtype=F64)
    q[..., 1] = 1.0
    k = torch.zeros(B, H, n, 64, dtype=F64)
    k[:, :, 1:, 1] = -0.99609375
    v = torch.zeros(B, H, n, 64, dtype=F64)
    v[:, :, 0] = (1 + torch.rand(B, H, 64, generator=g, dtype=F64)) * torch.sign(torch.randn(B, H, 64, generator=g, dtype=F64))
    v = v.to(torch.bfloat16)
    l = 1.0 + (n - 1) * 2.0 ** -0.99609375
    ref = (v[:, :, 0].to(F64) / l)[:, :, None].expand(B, H, n, 64).permute(0, 2, 1, 3).reshape(B, n, H * 64)
    return q.to(torch.bfloat16), k.to(torch.bfloat16), v, ref


def emulate_attention(q, k, v, mask_extra: int = 0, skip_alpha: bool = False, l_after_round: bool = False) -> torch.Tensor:
    """The kernel's online softmax in fp32 on the CPU, 128 keys per step: masked tail, running maximum, alpha rescale, P rounded
    to bf16 for P.V, l from the unrounded values, out = bf16(O * (1 / l)).  The flags seed mistakes: `mask_extra` more keys kept
    in the ragged last tile (they read as zero, as the TMA fill), no rescale of O, l summed after rounding."""
    q, k, v = q.float(), k.float(), v.float()
    B, H, nq, D = q.shape
    nkv = k.shape[2]
    ntiles = (nkv + 127) // 128
    pad = ntiles * 128 - nkv
    kp = torch.cat([k, k.new_zeros(B, H, pad, D)], 2)
    vp = torch.cat([v, v.new_zeros(B, H, pad, D)], 2)
    m = torch.full((B, H, nq, 1), -torch.inf)
    l = torch.zeros(B, H, nq, 1)
    o = torch.zeros(B, H, nq, D)
    for j in range(ntiles):
        kt, vt = kp[:, :, 128 * j:128 * (j + 1)], vp[:, :, 128 * j:128 * (j + 1)]
        s = q @ kt.transpose(-1, -2)
        valid = min(128, nkv - 128 * j) + (mask_extra if j == ntiles - 1 else 0)
        s[..., valid:] = -torch.inf
        m_new = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp2(m - m_new)
        e = torch.exp2(s - m_new)
        pb = e.to(torch.bfloat16).float()
        l = l * alpha + (pb if l_after_round else e).sum(-1, keepdim=True)
        o = (o if skip_alpha else o * alpha) + pb @ vt
        m = m_new
    out = (o * (1.0 / l)).to(torch.bfloat16)
    return out.permute(0, 2, 1, 3).reshape(B, nq, H * D)


# ----------------------------------------------------------------------------------------------- LayerNorm
def layernorm_ref(x, w=None, b=None, eps: float = 1e-5, out_dtype=torch.bfloat16):
    """LayerNorm over the last dim: (ref fp64, bound fp64).  The bound follows the kernel's fp32 steps: a per-lane sum of C/32
    values then 5 butterfly levels for the mean and for the variance, rsqrtf, the affine FMA and the store."""
    x = x.to(F64)
    C = x.shape[-1]
    mean = x.mean(-1, keepdim=True)
    d = x - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = d * rstd
    n_add = C / 32 + 6
    e_mean = n_add * EPS32 * x.abs().mean(-1, keepdim=True) * 2
    rel_r = 0.5 * e_mean ** 2 / (var + eps) + n_add * EPS32 * 2 + 2.0 ** -21
    exh = rstd * (e_mean + 2 * EPS32 * d.abs()) + xh.abs() * rel_r
    if w is not None:
        w, b = w.to(F64), b.to(F64)
        ref = xh * w + b
        e = exh * w.abs() + 2 * EPS32 * ref.abs()
    else:
        ref, e = xh, exh
    return ref, e + (ulp(ref, out_dtype) if out_dtype != torch.float32 else EPS32 * ref.abs())


# ----------------------------------------------------------------------------------------------- camera head
# The runtime rounds seven intermediates to bf16.  Where its fp32 value and the fp64 restatement's sit on opposite sides of a bf16
# rounding point, the two differ by one bf16 ulp there, and that difference propagates.  CAM_TOL bounds the result, as a fraction
# of the largest |output| of the call (camera_error).  An fp32 emulation with the same roundings measures up to 3.7e-3 at
# D = 256 (tests/test_kernel_ref_cpu.py); an attention scale of 1 / head_dim instead of 1 / sqrt(head_dim) gives 6e-2 and more.
CAM_TOL = 1e-2


def camera_error(out: torch.Tensor, ref: torch.Tensor) -> float:
    """max |out - ref| / max |ref| over all iterations, rows and the 9 pose values."""
    out, ref = out.to(F64).cpu(), ref.to(F64).cpu()
    if not torch.isfinite(out).all():
        return math.inf
    return float((out - ref).abs().max() / ref.abs().max())


def camera_ref(w: Dict[str, object], tokens: torch.Tensor, B: int, S: int, heads: int, iters: int = 4,
               dtype: torch.dtype = F64, attn_scale: Optional[float] = None) -> torch.Tensor:
    """The camera head (reference heads/camera_head.py:83-154) computed in `dtype`, rounding to bf16 exactly where the runtime
    stores bf16 (e, mod, xn, qkv, o, hid and g of its workspace).  w: the packed weights (Engine.cam: trunk blocks, tn_w, tn_b,
    rn_w, rn_b, empty, ew, eb, mw, mb, f1w, f1b, f2w, f2b).  tokens fp32 [B*S, D] -> activated poses [iters, B*S, 9].
    attn_scale replaces 1/sqrt(head_dim) (a seeded mistake)."""
    def t(x):
        return x.detach().to(dtype).cpu()

    def bf(x):
        return x.to(torch.bfloat16).to(dtype)

    def ln(x, wt=None, bb=None, eps=1e-5):
        mu = x.mean(-1, keepdim=True)
        d = x - mu
        y = d / torch.sqrt((d * d).mean(-1, keepdim=True) + eps)
        return y if wt is None else y * t(wt) + t(bb)

    def lin(x, wt, bb):
        return x @ t(wt).t() + t(bb)

    K, D = tokens.shape
    hd = D // heads
    scale = 1.0 / math.sqrt(hd) if attn_scale is None else attn_scale
    tok = ln(t(tokens), w["tn_w"], w["tn_b"])
    pose = None
    outs = []
    for it in range(iters):
        x = t(w["empty"])[None].expand(K, 9) if pose is None else pose
        e = lin(x, w["ew"], w["eb"])
        e = bf(e * torch.sigmoid(e))
        mod = bf(lin(e, w["mw"], w["mb"]))
        shift, sc, gate = mod[:, :D], mod[:, D:2 * D], mod[:, 2 * D:]
        h = gate * (ln(tok, eps=1e-6) * (1 + sc) + shift) + tok
        for blk in w["trunk"]:
            xn = bf(ln(h, blk.ln1_w, blk.ln1_b))
            qkv = bf(lin(xn, blk.w_qkv, blk.b_qkv)).reshape(B, S, 3, heads, hd)
            q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))          # [B, heads, S, hd]
            a = torch.softmax((q * scale) @ k.transpose(-1, -2), -1) @ v
            o = bf(a.permute(0, 2, 1, 3).reshape(K, D))
            h = h + t(blk.g1) * lin(o, blk.w_proj, blk.b_proj)
            xn = bf(ln(h, blk.ln2_w, blk.ln2_b))
            hid = bf(gelu(lin(xn, blk.w_fc1, blk.b_fc1)))
            h = h + t(blk.g2) * lin(hid, blk.w_fc2, blk.b_fc2)
        xn = bf(ln(h, w["rn_w"], w["rn_b"]))
        g = bf(gelu(lin(xn, w["f1w"], w["f1b"])))
        delta = lin(g, w["f2w"], w["f2b"])
        pose = delta if pose is None else pose + delta
        act = pose.clone()
        act[:, 7:] = act[:, 7:].clamp(min=0)
        outs.append(act)
    return torch.stack(outs)


# ----------------------------------------------------------------------------------------------- bilinear upsampling, DPT tail
# The resize kernels (ovg_upsample_bilinear's two kernels and the producer warps of the fused tail) compute the sample positions
# in fp32 and blend in fp32.  The references take the positions exactly as the kernels do (sample_positions) and blend in fp64, so
# what is left to bound is the blend:
#   * every output is a sum of four terms w_y w_x v, and each term passes through at most four fp32 roundings on any of the
#     kernels' evaluation orders (vertical then horizontal, horizontal then vertical, with or without FMA contraction):
#     BLEND_ROUNDINGS * EPS32 * sum |w v| (second-order terms are below 2^-40 of it);
#   * nvcc may contract w1 = fp32(s o) - i0 into fma(s, o, -i0), which moves w1 and w0 = 1 - w1 by up to EPS32 (|f| + 3):
#     position_slack.
BLEND_ROUNDINGS = 4.0001
# tail_tables_kernel: one table entry is four fp32 FMA chains of <= 144 terms, then two adds: <= 146 roundings of a partial sum.
TABLE_ROUNDINGS = 146


def sample_positions(n_src: int, n_dst: int):
    """align_corners sample positions as the kernels compute them: s = fp32(n_src - 1) / fp32(n_dst - 1), f = fp32(s o),
    i0 = int(f), i1 = i0 + (i0 < n_src - 1), w1 = f - i0 (exact), w0 = fp32(1 - w1).  Returns (i0, i1, w0, w1, f); the weights
    and f as fp64 [n_dst]."""
    if n_dst > 1:
        s = torch.tensor(float(n_src - 1), dtype=F32) / torch.tensor(float(n_dst - 1), dtype=F32)
    else:
        s = torch.tensor(0.0, dtype=F32)
    f = s * torch.arange(n_dst, dtype=F32)
    i0 = f.to(torch.int64)
    i1 = i0 + (i0 < n_src - 1).to(torch.int64)
    w1 = f - i0.to(F32)
    w0 = 1.0 - w1
    return i0, i1, w0.to(F64), w1.to(F64), f.to(F64)


def _blend(src: torch.Tensor, H: int, W: int):
    """fp64 bilinear blend of src [F, h, w, C] at the kernels' fp32 positions: (value, the fp32 blend's error bound, sum |w v|),
    all [F, H, W, C]."""
    Fr, h, w, C = src.shape
    dev = src.device
    yi0, yi1, wy0, wy1, fy = (t.to(dev) for t in sample_positions(h, H))
    xi0, xi1, wx0, wx1, fx = (t.to(dev) for t in sample_positions(w, W))
    s = src.to(F64)
    a, b = s[:, yi0], s[:, yi1]                                                  # [F, H, w, C]
    cy = lambda t: t[None, :, None, None]                                        # noqa: E731
    cx = lambda t: t[None, None, :, None]                                        # noqa: E731
    r = cy(wy0) * a + cy(wy1) * b
    value = cx(wx0) * r[:, :, xi0] + cx(wx1) * r[:, :, xi1]
    del r
    ar = cy(wy0) * a.abs() + cy(wy1) * b.abs()
    absum = cx(wx0) * ar[:, :, xi0] + cx(wx1) * ar[:, :, xi1]
    slack = EPS32 * (cx(fx.abs()) + 3) * (ar[:, :, xi0] + ar[:, :, xi1])
    del ar
    bb = a.abs() + b.abs()
    slack += EPS32 * (cy(fy.abs()) + 3) * (cx(wx0) * bb[:, :, xi0] + cx(wx1) * bb[:, :, xi1])
    return value, BLEND_ROUNDINGS * EPS32 * absum + slack, absum


def embedding_map(tx: Optional[torch.Tensor], ty: Optional[torch.Tensor], H: int, W: int, C: int, device=None) -> torch.Tensor:
    """The separable position embedding as a map fp64 [H, W, C]: channels [0, C/2) = tx[x], [C/2, C) = ty[y] (zeros without)."""
    if tx is None:
        return torch.zeros(H, W, C, dtype=F64, device=device)
    tx, ty = tx.to(device=device, dtype=F64), ty.to(device=device, dtype=F64)
    return torch.cat([tx[None].expand(H, W, C // 2), ty[:, None].expand(H, W, C // 2)], -1)


def bilinear_ref(src, H: int, W: int, tx=None, ty=None, dtype=torch.bfloat16):
    """ovg_upsample_bilinear on the interior src [F, h, w, C] (align_corners resize + the separable table): (ref fp64
    [F, H, W, C], bound).  The bound is one ulp of the 16-bit store plus the fp32 blend and the table add."""
    value, err, absum = _blend(src, H, W)
    emb = embedding_map(tx, ty, H, W, src.shape[-1], src.device)[None]
    ref = value + emb
    bound = ulp(ref, dtype) + err + EPS32 * (absum + emb.abs())
    return ref, bound


def upsample_path(w: int, C: int) -> str:
    """Which kernel ovg_upsample_bilinear launches, restated from its launch rule: "rows" (two-pass, one source row of 32 channels
    in 48 KB of shared memory) when C % 32 == 0 and w * 128 B <= 48 KB, else "direct"."""
    return "rows" if C % 32 == 0 and w * 32 * 4 <= 48 * 1024 and C // 32 <= 65535 else "direct"


def conv3x3(x: torch.Tensor, wk: torch.Tensor) -> torch.Tensor:
    """3x3 convolution with zero padding, NHWC: x [F, H, W, C], wk [O, 3, 3, C] -> [F, H, W, O] (fp64, as nine matmuls)."""
    Fr, H, W, C = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    out = torch.zeros(Fr, H, W, wk.shape[0], dtype=x.dtype, device=x.device)
    for ky in range(3):
        for kx in range(3):
            out += xp[:, ky:ky + H, kx:kx + W] @ wk[:, ky, kx].t()
    return out


ROW_CLASSES = ((1, 2), (0, 2), (0, 1))     # kernel taps of the other axis inside the image: first, interior, last row / column


def tail_tables_ref(tx, ty, w3x3, H: int, W: int):
    """tail_tables_kernel: the position embedding's image under the 3x3 kernel, split by linearity into gx [3, W, 32] (class =
    the output row's: 0 first row, 1 interior, 2 last row; x half of the embedding) and gy [3, H, 32] (class = the output
    column's; y half), so that conv(E)[y, x] = gx[rc(y), x] + gy[cc(x), y].  w3x3 [32, 9 * 128] in K order (ky, kx, c)."""
    wk = w3x3.to(F64).reshape(32, 3, 3, 128)
    out = []
    for t, n, part in ((tx, W, 0), (ty, H, 1)):
        tp = torch.nn.functional.pad(t.to(device=wk.device, dtype=F64), (0, 0, 1, 1))
        g = torch.zeros(3, n, 32, dtype=F64, device=wk.device)
        for cls, (lo, hi) in enumerate(ROW_CLASSES):
            for ks in range(3):                                   # tap along the table's own axis
                ws = sum((wk[:, ko, ks, :64] if part == 0 else wk[:, ks, ko, 64:]) for ko in range(lo, hi + 1))
                g[cls] += tp[ks:ks + n] @ ws.t()
        out.append(g)
    return out[0], out[1]


def dpt_tail_ref(src, tx, ty, w3x3, bias, w2, b2, head_act: int, H: int, W: int, dtype=torch.bfloat16):
    """ovg_dpt_tail on the interior src [F, h, w, 128]: resize -> 16-bit operand -> + embedding -> 3x3 conv 128 -> 32 + bias ->
    ReLU -> 1x1 -> activations.  Returns (preds [F, H, W, outc-1], conf [F, H, W], bound of preds, bound of conf), fp64.

    The producers round the fp32 blend to 16 bits; the reference uses round(up64) as the conv operand and allows the
    neighbouring 16-bit value only where up64 lies within the blend's error bound of a rounding point.  The embedding enters
    in fp32 through the tables.  Pre-activation bound: tensor-core accumulation over K = 9 * 128, the two fp32 adds that join
    the three kernel rows' partial sums, the operand flips, the tables' fp32 FMA chains and the three epilogue adds."""
    dev = src.device
    up, err, _ = _blend(src, H, W)
    op = round_to(up, dtype)
    dop = torch.maximum((round_to(up + err, dtype) - op).abs(), (round_to(up - err, dtype) - op).abs())
    del up, err
    wk = w3x3.to(device=dev, dtype=F64).reshape(32, 3, 3, 128)
    wa = wk.abs()
    emb = embedding_map(tx, ty, H, W, 128, dev)[None]
    h = conv3x3(op + emb, wk) + bias.to(device=dev, dtype=F64)
    absacc = conv3x3(op.abs(), wa)
    flips = conv3x3(dop, wa)
    del op, dop
    abse = conv3x3(emb.abs(), wa) if tx is not None else torch.zeros_like(absacc[:1])
    eh = acc_bound(absacc, 9 * 128) + 2 * EPS32 * absacc + flips + TABLE_ROUNDINGS * EPS32 * abse \
        + 3 * EPS32 * (absacc + bias.to(device=dev, dtype=F64).abs() + abse)
    return head_post(h, eh, w2, b2, head_act)


# ----------------------------------------------------------------------------------------------- fused tail geometry
FT_VBUF_PX = 80          # source pixels a 130-pixel strip may span (tail.cuh): the ring row and itab size


def tail_supported(h: int, w: int, H: int, W: int, C: int = 128) -> bool:
    """ovg_dpt_tail_supported, restated in fp32."""
    import numpy as np
    if C != 128 or h < 2 or w < 2 or H < h or W < w:
        return False
    sx = np.float32(w - 1) / np.float32(W - 1)
    return int(sx * np.float32(129.0)) + 3 <= FT_VBUF_PX


def tail_schedule(F: int, H: int, W: int, sms: int) -> Dict[str, int]:
    """ovg_dpt_tail's work split on a device with `sms` SMs: 128-pixel strips, segments of seg_rows output rows (two halo rows
    each), about three work items per SM."""
    n_strips = (W + 127) // 128
    segs = max(1, (3 * sms + F * n_strips - 1) // (F * n_strips))
    segs = min(segs, H)
    seg_rows = (H + segs - 1) // segs
    if seg_rows < 8 and H >= 8:
        seg_rows = 8
    n_segs = (H + seg_rows - 1) // seg_rows
    return dict(n_strips=n_strips, seg_rows=seg_rows, n_segs=n_segs, n_items=F * n_strips * n_segs,
                last_strip_px=W - 128 * (n_strips - 1))


def tail_strip(w: int, W: int, strip: int):
    """The producer's walk for one strip, in fp32 as tail.cuh: (x_lo, x_hi, xs_lo, ns, itab) with itab a list of
    (first strip row, pixel count) per source interval xs_lo + j, j < ns."""
    import numpy as np
    sx = np.float32(w - 1) / np.float32(W - 1)
    x0 = 128 * strip
    x_lo, x_hi = max(x0 - 1, 0), min(x0 + 128, W - 1)
    fl = lambda X: int(sx * np.float32(X))                                     # noqa: E731
    xs_lo = fl(x_lo)
    xs_hi = min(fl(x_hi) + 1, w - 1)
    ns = xs_hi - xs_lo + 1
    itab = []
    for j in range(ns):
        sabs = xs_lo + j
        Xg = max(int(np.float32(sabs) / sx) - 2, x_lo)
        while Xg <= x_hi and fl(Xg) < sabs:
            Xg += 1
        n = 0
        while Xg + n <= x_hi and fl(Xg + n) == sabs:
            n += 1
        itab.append((Xg - (x0 - 1), n))
    return x_lo, x_hi, xs_lo, ns, itab


# ----------------------------------------------------------------------------------------------- im2col of the patch embeddings
def image_cols_ref(images: torch.Tensor, mean3, std3, patch: int, ldc: int) -> torch.Tensor:
    """ovg_image_im2col in fp32 on the CPU: (v - mean) * istd with istd = 1 / std rounded to fp32 (the host's 1.0f / std), stored
    as bf16 rows (k, py, px) x columns (c, ky, kx), zero-padded to ldc.  Two IEEE roundings and no contraction opportunity,
    so this is bit-exact."""
    K, _, H, W = images.shape
    hp, wp = H // patch, W // patch
    mean = torch.tensor([float(v) for v in mean3], dtype=F32)[None, :, None, None]
    istd = (1.0 / torch.tensor([float(v) for v in std3], dtype=F32))[None, :, None, None]
    v = (images.to(F32).cpu() - mean) * istd
    cols = v.reshape(K, 3, hp, patch, wp, patch).permute(0, 2, 4, 1, 3, 5).reshape(K * hp * wp, 3 * patch * patch)
    out = torch.zeros(K * hp * wp, ldc, dtype=torch.bfloat16)
    out[:, :3 * patch * patch] = cols.to(torch.bfloat16)
    return out


def depth_scale_ref(depth: torch.Tensor, mask: torch.Tensor, idx_stats: Sequence[int]) -> torch.Tensor:
    """The per-scene scale of ovg_depth_im2col from exact sums: fp32(1 / (fp32(sum / count) + 1e-8f)), 0 without a valid pixel
    (fp32 [B]).  Equal to the kernel's bit for bit when its fp32 partial sums are exact (dyadic depths)."""
    d = depth.to(F64).cpu()[:, list(idx_stats)]
    m = mask.cpu()[:, list(idx_stats)] > 0
    out = torch.zeros(d.shape[0], dtype=F32)
    for b in range(d.shape[0]):
        cnt = int(m[b].sum())
        if cnt:
            mean = torch.tensor(float(d[b][m[b]].sum()) / cnt, dtype=F64).to(F32)
            out[b] = torch.tensor(1.0, dtype=F32) / (mean + torch.tensor(1e-8, dtype=F32))
    return out


def depth_cols_ref(depth: torch.Tensor, mask: torch.Tensor, scale: torch.Tensor, idx_cols: Sequence[int], patch: int):
    """ovg_depth_im2col's rows for the views idx_cols, given the per-scene fp32 scale: [d * scale * m, m] in fp32 ((d * scale)
    rounded, then * m; no contraction opportunity), stored as bf16 rows (b, view, py, px) x columns (ky, kx) of each half."""
    d = depth.to(F32).cpu()[:, list(idx_cols)]
    m = mask.to(F32).cpu()[:, list(idx_cols)]
    B, S, H, W = d.shape
    hp, wp = H // patch, W // patch
    v = (d * scale.to(F32).cpu()[:, None, None, None]) * m

    def unfold(t):
        return t.reshape(B, S, hp, patch, wp, patch).permute(0, 1, 2, 4, 3, 5).reshape(B * S * hp * wp, patch * patch)
    return torch.cat([unfold(v), unfold(m)], 1).to(torch.bfloat16)
