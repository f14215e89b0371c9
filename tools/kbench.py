"""Kernel micro-benchmarks at the cfg2 shapes (B=1, S=8, 518^2): CUDA-event timing, L2 flushed between iterations."""
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


res = {}
KB = os.environ.get("KB", "all")
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
os.makedirs("gpurun_out", exist_ok=True)
json.dump(res, open("gpurun_out/kbench.json", "w"), indent=1)
