"""DPT output tail at the product shape (8 frames, 296^2 -> 518^2, 128 channels): the fused kernel (ovg_dpt_tail), next to the
two-kernel composition it replaced, ovg_upsample_bilinear + the generic gemm_kernel<32, EPI_HEADTAIL> (GPU box).  The model takes
the fused kernel at this shape; the two-kernel leg is a point of comparison, not a path the product runs."""
import json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from omnivggt_official_b200 import ops

dev = torch.device("cuda", 0)
Fr, h, w, H, W, Cin = 8, 296, 296, 518, 518, 128
dt = torch.float16
flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)


def timeit(fn, iters=10):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2] * 1e3


res = {"tag": sys.argv[1] if len(sys.argv) > 1 else ""}
for outc, act in ((2, 0), (4, 1)):
    xp = torch.zeros(Fr, h + 2, w + 2, Cin, device=dev, dtype=dt)
    xp[:, 1:-1, 1:-1] = torch.randn(Fr, h, w, Cin, device=dev).to(dt)
    wb = (torch.randn(32, 9 * Cin, device=dev) * (9 * Cin) ** -0.5).to(dt)
    b1, w2, b2 = torch.randn(32, device=dev) * 0.1, torch.randn(outc, 32, device=dev) * 32 ** -0.5, torch.randn(outc, device=dev) * 0.1
    tx, ty = torch.randn(W, 64, device=dev) * 0.1, torch.randn(H, 64, device=dev) * 0.1
    res[f"fused_outc{outc}_us"] = timeit(lambda: ops.dpt_tail(xp, tx, ty, wb, b1, w2, b2, act, Fr, h, w, H, W))
    dst = torch.zeros(Fr, H + 2, W + 2, Cin, device=dev, dtype=dt)
    p2 = torch.zeros(Fr, H, W, outc - 1, device=dev)
    c2 = torch.zeros(Fr, H, W, device=dev)
    taps = [(ky - 1) * (W + 2) + (kx - 1) for ky in range(3) for kx in range(3)]

    def two():
        ops.upsample_bilinear(xp, dst, tx, ty, Fr, h, w, H, W, Cin)
        ops.gemm(dst.reshape(-1, Cin), wb, taps=taps, epi=ops.L.EPI_HEADTAIL, bias=b1, w2=w2, b2=b2, outc=outc, head_act=act,
                 preds=p2, conf=c2, rowmap=ops.L.ROWS_PAD, gh=H, gw=W)
    res[f"two_kernels_outc{outc}_us"] = timeit(two)
print(json.dumps(res))
