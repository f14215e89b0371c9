"""Attention micro-benchmark: the three shapes the model runs (global 8 views, frame, global 24 views) with CUDA-event timing
and an L2 flush between iterations, torch SDPA (library kernel) beside it.  OVG_LIB_PATH selects an A/B build of libovg.

    python tools/attn_bench.py [tag]            -> one JSON line
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from omnivggt_official_b200 import ops  # noqa: E402

BF16 = torch.bfloat16
flush_buf = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=7, warm=2):
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


res = {"tag": sys.argv[1] if len(sys.argv) > 1 else "", "lib": os.environ.get("OVG_LIB_PATH", "libovg.so"),
       "split_tail": os.environ.get("ATTN_SPLIT", "1") != "0"}
shapes = {"global8": (1, 16, 8 * 1374), "frame8": (8, 16, 1374), "global24": (1, 16, 24 * 1374), "global4": (1, 16, 4 * 1374)}
scratch = ops.attention_scratch("cuda") if os.environ.get("ATTN_SPLIT", "1") != "0" else None     # KV-split tail tiles (ovg_attention scratch)
if os.environ.get("ATTN_SHAPES"):
    shapes = {k: shapes[k] for k in os.environ["ATTN_SHAPES"].split(",")}
for name, (b, h, n) in shapes.items():
    g = torch.Generator(device="cuda").manual_seed(1)
    q = (torch.randn(b, h, n, 64, device="cuda", generator=g) * 0.18).to(BF16)
    k = torch.randn(b, h, n, 64, device="cuda", generator=g).to(BF16)
    v = torch.randn(b, h, n, 64, device="cuda", generator=g).to(BF16)
    o = torch.empty(b, n, h * 64, device="cuda", dtype=BF16)
    ms = timeit(lambda: ops.attention(q, k, v, o, b, h, n, scratch=scratch), iters=5 if n > 20000 else 7)
    fl = 4.0 * b * h * n * n * 64
    res[name] = dict(ms=round(ms, 4), tflops=round(fl / ms / 1e9, 1))
    if os.environ.get("ATTN_SDPA", "1") != "0":
        ms2 = timeit(lambda: F.scaled_dot_product_attention(q, k, v, scale=0.125), iters=5 if n > 20000 else 7)
        res[name]["sdpa_ms"] = round(ms2, 4)
        # value check against the library kernel (q carries log2(e)/8; SDPA gets the matching natural-log scale)
        ref = F.scaled_dot_product_attention(q.float() if n < 3000 else q, k.float() if n < 3000 else k,
                                             v.float() if n < 3000 else v, scale=0.6931471805599453).transpose(1, 2).reshape(b, n, h * 64)
        ops.attention(q, k, v, o, b, h, n, scratch=scratch)
        torch.cuda.synchronize()
        res[name]["rel_l2_vs_sdpa"] = round(((o.float() - ref.float()).norm() / ref.float().norm()).item(), 5)
        o2 = torch.empty_like(o)
        ops.attention(q, k, v, o2, b, h, n, scratch=scratch)
        torch.cuda.synchronize()
        res[name]["bit_identical_rerun"] = bool(torch.equal(o, o2))
print(json.dumps(res))
