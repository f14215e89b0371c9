"""Kernel micro-benchmarks at the cfg2 shapes (B=1, S=8, 518^2): CUDA-event timing, L2 flushed between iterations.

KB=gemm runs only the hot-path GEMMs with their real epilogues at S = 8 and 24 (hot_gemms), KB=attn only attention; KB_OUT sets
the JSON file the results go to."""
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from omnivggt_official_b200 import ops  # noqa: E402

BF16 = torch.bfloat16
dev = "cuda"
flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush_buf.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def timeit_launches(fn, launches=40, warm=5):
    """ms per launch: CUDA events around `launches` back-to-back launches (no flush: in a forward the weights and often the
    activations of a GEMM are still in L2 from the op before)."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / launches


def card():
    """Name, power limit and SM clocks of device 0, read (never set) through nvidia-smi."""
    import subprocess
    d = dict(name=torch.cuda.get_device_name(0))
    try:
        q = "power.limit,clocks.sm,clocks.max.sm"
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        d.update(zip(("power_limit_w", "sm_clock_mhz", "sm_clock_max_mhz"), (v.strip() for v in r.stdout.split(","))))
    except Exception as ex:  # the numbers are still valid without it, just less well labelled
        d["nvidia_smi"] = repr(ex)
    return d


def hot_gemms(res):
    """The GEMMs of the transformer blocks and the DPT 3x3 conv with their real epilogues, as the forward runs them (block_n
    chosen by the library), at S = 8 (cfg2) and S = 24 (cfg5) views of 1374 tokens, next to cuBLAS on the same shape."""
    C = 1024
    for S in (8, 24):
        M = S * 1374
        a = torch.randn(M, 4 * C, device=dev).to(BF16)
        x = torch.randn(M, C, device=dev).to(BF16)
        w = {(n, k): (torch.randn(n, k, device=dev) * k ** -0.5).to(BF16) for n, k in ((3 * C, C), (C, C), (4 * C, C), (C, 4 * C))}
        bias = torch.randn(4 * C, device=dev) * 0.1
        gamma = torch.randn(C, device=dev) * 0.1
        xres = torch.randn(M, C, device=dev)
        h = torch.empty(M, 4 * C, device=dev, dtype=BF16)
        ln = [torch.ones(64, device=dev), torch.zeros(64, device=dev), torch.ones(64, device=dev), torch.zeros(64, device=dev)]
        cos, sin = ops.rope_tables(38, dev)
        q = torch.empty(1, 16, M, 64, device=dev, dtype=BF16)
        k, v = torch.empty_like(q), torch.empty_like(q)
        cases = {
            "qkv_ln_rope": (3 * C, C, lambda: ops.qkv_proj(x, w[3 * C, C], bias[:3 * C], *ln, q, k, v, ntok=M, T=1374, nspecial=5,
                                                           wp=37, rope_cos=cos, rope_sin=sin), x, w[3 * C, C]),
            "proj_resid": (C, C, lambda: ops.linear_resid(x, w[C, C], bias[:C], gamma, xres), x, w[C, C]),
            "fc1_gelu": (4 * C, C, lambda: ops.linear_bf16(x, w[4 * C, C], bias, act=ops.L.ACT_GELU, out=h), x, w[4 * C, C]),
            "fc2_resid": (C, 4 * C, lambda: ops.linear_resid(a, w[C, 4 * C], bias[:C], gamma, xres), a, w[C, 4 * C]),
        }
        for name, (N, K, fn, ca, cb) in cases.items():
            ms = timeit_launches(fn)
            ms_cublas = timeit_launches(lambda: torch.matmul(ca, cb.t()))
            fl = 2 * M * N * K
            res[f"hot_{name}_S{S}"] = dict(M=M, N=N, K=K, ms=ms, tflops=fl / ms / 1e9, cublas_ms=ms_cublas,
                                           cublas_tflops=fl / ms_cublas / 1e9)
        del a, x, w, xres, h, q, k, v
        # DPT 3x3 conv 256 -> 256 at the 1/4-resolution level (S frames x 148^2): ROWS_PAD, 9 taps, bias, ReLU, two skips
        hh = ww = 148
        xp = torch.zeros(S, hh + 2, ww + 2, 256, device=dev, dtype=BF16)
        xp[:, 1:-1, 1:-1] = torch.randn(S, hh, ww, 256, device=dev).to(BF16)
        flat = xp.reshape(-1, 256)
        wc = (torch.randn(256, 9 * 256, device=dev) * (9 * 256) ** -0.5).to(BF16)
        sk1, sk2, outp = torch.randn_like(xp), torch.randn_like(xp), torch.empty_like(xp)
        taps = [(ky - 1) * (ww + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
        b256 = torch.randn(256, device=dev)
        ms = timeit_launches(lambda: ops.gemm(flat, wc, taps=taps, epi=ops.L.EPI_BF16, bias=b256, act=ops.L.ACT_RELU, out=outp, ldo=256,
                                              skip1=sk1, skip2=sk2, rowmap=ops.L.ROWS_PAD, gh=hh, gw=ww), launches=20)
        # cuBLAS on the same FLOPs: [rows, 9 * 256] x [9 * 256, 256] (an im2col the conv does not need to materialise)
        acol = torch.randn(flat.shape[0], 9 * 256, device=dev).to(BF16)
        ms_cublas = timeit_launches(lambda: torch.matmul(acol, wc.t()), launches=20)
        fl = 2 * flat.shape[0] * 256 * 9 * 256
        res[f"hot_conv3x3_pad_skips_S{S}"] = dict(M=flat.shape[0], N=256, K=9 * 256, ms=ms, tflops=fl / ms / 1e9, cublas_ms=ms_cublas,
                                                  cublas_tflops=fl / ms_cublas / 1e9)
        del xp, flat, sk1, sk2, outp, acol
        torch.cuda.empty_cache()


res = {}
KB = os.environ.get("KB", "all")
OUT = os.environ.get("KB_OUT", os.path.join("build_ab", "kbench.json"))
res["card"] = card()
if KB in ("all", "gemm"):
    hot_gemms(res)
if KB == "gemm":
    for k_, v_ in res.items():
        print(k_, json.dumps(v_))
    os.makedirs(os.path.dirname(OUT) or ".", exist_ok=True)
    json.dump(res, open(OUT, "w"), indent=1)
    sys.exit(0)
S, T, C = int(os.environ.get("S", 8)), 1374, 1024
M = S * T
a = torch.randn(M, C, device=dev).to(BF16)
for name, N, K, bns in () if KB == "attn" else (("qkv", 3072, 1024, (64, 128)), ("proj", 1024, 1024, (64, 128)), ("fc1", 4096, 1024, (64, 128)), ("fc2", 1024, 4096, (64, 128))):
    x = torch.randn(M, K, device=dev).to(BF16)
    w = (torch.randn(N, K, device=dev) * K ** -0.5).to(BF16)
    bias = torch.randn(N, device=dev)
    out = torch.empty(M, N, device=dev, dtype=BF16)
    xres = torch.randn(M, N, device=dev)
    gamma = torch.randn(N, device=dev)
    for bn in bns:
        if name in ("proj", "fc2"):
            ms = timeit(lambda: ops.linear_resid(x, w, bias, gamma, xres, block_n=bn))
        elif name == "fc1":
            ms = timeit(lambda: ops.linear_bf16(x, w, bias, act=ops.L.ACT_GELU, out=out, block_n=bn))
            ms0 = timeit(lambda: ops.linear_bf16(x, w, bias, out=out, block_n=bn))
            res[f"gemm_fc1_noact_bn{bn}"] = dict(ms=ms0, tflops=2 * M * N * K / ms0 / 1e9)
        else:
            ms = timeit(lambda: ops.linear_bf16(x, w, bias, out=out, block_n=bn))
        res[f"gemm_{name}_bn{bn}"] = dict(ms=ms, tflops=2 * M * N * K / ms / 1e9)
    ms = timeit(lambda: torch.matmul(x, w.t()))
    res[f"cublas_{name}"] = dict(ms=ms, tflops=2 * M * N * K / ms / 1e9)
# qkv epilogue
w = (torch.randn(3 * C, C, device=dev) * C ** -0.5).to(BF16)
bias = torch.randn(3 * C, device=dev)
ones, zeros = torch.ones(64, device=dev), torch.zeros(64, device=dev)
cos, sin = ops.rope_tables(38, dev)
q = torch.empty(1, 16, M, 64, device=dev, dtype=BF16)
k, v = torch.empty_like(q), torch.empty_like(q)
for bn in (64, 128) if KB != "attn" else (128,):
    ms = timeit(lambda: ops.qkv_proj(a, w, bias, ones, zeros, ones, zeros, q, k, v, ntok=M, T=T, nspecial=5, wp=37, rope_cos=cos, rope_sin=sin, block_n=bn))
    res[f"gemm_qkv_fused_bn{bn}"] = dict(ms=ms, tflops=2 * M * 3 * C * C / ms / 1e9)
# DPT-shaped 3x3 conv: 8 frames x 148^2, 256 -> 256
Fr, hh, ww = (8, 148, 148) if KB != "attn" else (1, 8, 8)
xp = torch.zeros(Fr, hh + 2, ww + 2, 256, device=dev, dtype=BF16)
xp[:, 1:-1, 1:-1] = torch.randn(Fr, hh, ww, 256, device=dev).to(BF16)
wc = (torch.randn(256, 9 * 256, device=dev) * (9 * 256) ** -0.5).to(BF16)
outp = torch.empty_like(xp)
taps = [(ky - 1) * (ww + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
bias256 = torch.randn(256, device=dev)
for bn in (64, 128) if KB != "attn" else ():
    ms = timeit(lambda: ops.gemm(xp.reshape(-1, 256), wc, taps=taps, epi=ops.L.EPI_BF16, bias=bias256, act=ops.L.ACT_RELU, out=outp, ldo=256, rowmap=ops.L.ROWS_PAD, gh=hh, gw=ww, block_n=bn), iters=5)
    res[f"conv3x3_148_bn{bn}"] = dict(ms=ms, tflops=2 * Fr * hh * ww * 256 * 256 * 9 / ms / 1e9)
# attention: global and frame
o = torch.empty(1, M, C, device=dev, dtype=BF16)
ms = timeit(lambda: ops.attention(q, k, v, o, 1, 16, M), iters=5)
res["attn_global"] = dict(ms=ms, tflops=4 * M * M * C / ms / 1e9)
qf, kf, vf = (t.reshape(16, S, T, 64).transpose(0, 1).contiguous() for t in (q, k, v))
ms = timeit(lambda: ops.attention(qf, kf, vf, o, S, 16, T))
res["attn_frame"] = dict(ms=ms, tflops=4 * S * T * T * C / ms / 1e9)
if KB != "attn":
    # DPT output_conv1-shaped conv: 8 frames x 296^2, 256 -> 128
    xq = torch.zeros(8, 298, 298, 256, device=dev, dtype=BF16)
    wq = (torch.randn(128, 9 * 256, device=dev) * (9 * 256) ** -0.5).to(BF16)
    oq = torch.empty(8, 298, 298, 128, device=dev, dtype=BF16)
    tq = [(ky - 1) * 298 + (kx - 1) for ky in range(3) for kx in range(3)]
    b128 = torch.randn(128, device=dev)
    for bn in (32, 64, 128):
        ms = timeit(lambda: ops.gemm(xq.reshape(-1, 256), wq, taps=tq, epi=ops.L.EPI_BF16, bias=b128, out=oq, ldo=128, rowmap=ops.L.ROWS_PAD, gh=296, gw=296, block_n=bn), iters=5)
        res[f"conv3x3_296_n128_bn{bn}"] = dict(ms=ms, tflops=2 * 8 * 296 * 296 * 256 * 128 * 9 / ms / 1e9)
    del xq, oq
import torch.nn.functional as F
ms = timeit(lambda: F.scaled_dot_product_attention(q, k, v), iters=5)
res["sdpa_global_torch"] = dict(ms=ms, tflops=4 * M * M * C / ms / 1e9)
# layernorm
x32 = torch.randn(M, C, device=dev)
ln_out = torch.empty(M, C, device=dev, dtype=BF16)
ln_w, ln_b = torch.ones(C, device=dev), torch.zeros(C, device=dev)
ms = timeit(lambda: ops.layernorm(x32, ln_out, ln_w, ln_b))
res["layernorm"] = dict(ms=ms, gbs=M * C * 6 / ms / 1e6)


def timeit_warm(fn, iters=20):
    for _ in range(3):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


g = torch.cuda.CUDAGraph()
ops.layernorm(x32, ln_out, ln_w, ln_b)
torch.cuda.synchronize()
with torch.cuda.graph(g):
    for _ in range(20):
        ops.layernorm(x32, ln_out, ln_w, ln_b)
ms = timeit_warm(g.replay, iters=5) / 20
res["layernorm_warm_l2"] = dict(ms=ms, gbs=M * C * 6 / ms / 1e6)
for k_, v_ in res.items():
    print(k_, json.dumps(v_))
os.makedirs(os.path.dirname(OUT) or ".", exist_ok=True)
json.dump(res, open(OUT, "w"), indent=1)
