"""What the DPT heads cost in a full-size forward, and what the fp32 layer export costs: the full model (synthetic weights) at
cfg2 (1 scene x 8 views @ 518^2, images only) and cfg5 (1 scene x 24 views @ 518^2, partial depth / camera aux).

Timed with CUDA events over --reps calls after a warm-up, per call:
  forward, all heads            (CUDA-graph replay, as bench.py runs it)
  forward, point_head = None    (the reference's --save_glb / viewer path reads depth only)
  forward, both DPT heads None  (pose only)
  model.aggregator(...)         (all 24 layers exported in fp32, eager: component calls are not graph captured)
  forward, all heads, eager     (the same launches as model.aggregator's, for comparison)
        python tools/heads_bench.py [--reps 10]"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (configs and seeded inputs only)
from tools.cloud_bench import power_limit  # noqa: E402

CONFIGS = ("cfg2", "cfg5")


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return round(t0.elapsed_time(t1) / reps, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT
    with torch.device("cuda"):
        m = OmniVGGT(init_seed=None)
    m.randomize_(0).eval()
    heads = {n: getattr(m, n) for n in ("depth_head", "point_head")}
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "configs": []}
    for name in CONFIGS:
        cfg = bench.CONFIGS[name]
        inp = {k: v.cuda() for k, v in bench.synth_inputs(1, cfg["S"], seed=0).items()}
        kw = dict(depth_gt_index=cfg["depth_idx"], camera_gt_index=cfg["cam_idx"])
        row = {"config": name, "views": cfg["S"]}
        m.use_cuda_graph = True
        row["forward_ms"] = timed(lambda: m(**inp, **kw), args.reps, 3)
        m.point_head = None
        row["forward_no_point_head_ms"] = timed(lambda: m(**inp, **kw), args.reps, 3)
        m.depth_head = None
        row["forward_pose_only_ms"] = timed(lambda: m(**inp, **kw), args.reps, 3)
        for n, h in heads.items():
            setattr(m, n, h)
        m.use_cuda_graph = False
        row["forward_eager_ms"] = timed(lambda: m(**inp, **kw), args.reps, 1)
        row["aggregator_fp32_layers_ms"] = timed(lambda: m.aggregator(**inp, **kw), args.reps, 1)
        torch.cuda.empty_cache()
        row["dpt_heads_share"] = round(1.0 - row["forward_pose_only_ms"] / row["forward_ms"], 3)
        row["point_head_share"] = round(1.0 - row["forward_no_point_head_ms"] / row["forward_ms"], 3)
        res["configs"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
