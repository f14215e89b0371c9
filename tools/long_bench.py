"""Long captures: OmniVGGT.reconstruct (view sets of --chunk views sharing --overlap, aligned and merged on the device) at
518 x 518 against one forward of all S views, and the alignment of one view-set boundary on its own.

Model: the full architecture with seeded random weights (no checkpoint offline), all heads.  Sizes: S = 48, 96 and 192 by
default.  reconstruct runs its forwards from one captured CUDA graph (every view set has the same signature); the single
forward of S views runs eagerly (its launch overhead is negligible at these sizes and a graph would double its memory), and
is skipped above --single-max views or reported as not fitting when it runs out of memory.  The boundary is what
reconstruct adds per view set after the forward and the decode (OmniVGGT._merge_view_set): the two confidence masks over the
shared views, the estimate (ovg_sim3_estimate), its statistics read back, the application to the new views
(ovg_sim3_apply) and the copies.
Every timing is CUDA events around calls that end in a device synchronise, after a warm-up of every shape; the median of
--reps.  The card's name and power limit are read in the same run.
        python tools/long_bench.py [--sizes 48 96 192] [--reps 3] [--single-max 192]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def _events(fn, reps):
    fn()                                            # warm-up of the shape
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[48, 96, 192])
    ap.add_argument("--chunk", type=int, default=24)
    ap.add_argument("--overlap", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--single-max", type=int, default=192)
    args = ap.parse_args()
    from omnivggt_official_b200 import OmniVGGT, ops
    from omnivggt_official_b200.model import chunk_schedule
    from oracle.synth import make_inputs
    H = W = 518
    with torch.device("cuda"):
        m = OmniVGGT(init_seed=None)
    m.randomize_(0).eval()
    info = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    print(json.dumps(info), flush=True)
    rows = []
    for S in args.sizes:
        images = make_inputs(1, S, H, W, seed=S)["images"].cuda()
        chunks = chunk_schedule(S, args.chunk, args.overlap)
        m.use_cuda_graph = True
        m.reconstruct(images, chunk=args.chunk, overlap=args.overlap)       # the first calls capture the graph
        rec_ms = _events(lambda: m.reconstruct(images, chunk=args.chunk, overlap=args.overlap), args.reps)
        row = {"S": S, "chunk": args.chunk, "overlap": args.overlap, "view_sets": len(chunks),
               "views_run": sum(b - a for a, b in chunks), "reconstruct_ms": round(rec_ms, 1),
               "reconstruct_ms_per_view": round(rec_ms / S, 2)}
        # one boundary on its own: the second view set against the merge of the first
        out = m.reconstruct(images[:, :chunks[1][1]], chunk=args.chunk, overlap=args.overlap)
        (a, b), n0 = chunks[1], chunks[0][1]
        merged = {k: v.clone() for k, v in out.items() if torch.is_tensor(v) and k not in ("images", "sim3", "align_pairs",
                                                                                            "align_rmse")}
        raw = m(images[:, a:b])
        ext, intr, c2w = ops.pose_decode(raw["pose_enc"][0].float().contiguous(), H, W)
        r = {"extrinsic": ext, "intrinsic": intr, "depth": raw["depth"][0], "depth_conf": raw["depth_conf"][0],
             "world_points": raw["world_points"][0], "world_points_conf": raw["world_points_conf"][0],
             "world_points_from_depth": ops.unproject_depth(raw["depth"][0].float().reshape(b - a, H, W), intr, c2w, H, W)}
        del raw, out
        row["boundary_ms"] = round(_events(lambda: OmniVGGT._merge_view_set(merged, r, 1, a, n0, b, "depth", 50.0),
                                           max(args.reps, 5)), 3)
        row["boundary_shared_views"], row["boundary_new_views"] = n0 - a, b - n0
        del merged, r
        torch.cuda.empty_cache()
        if S <= args.single_max:
            m.use_cuda_graph = False
            try:
                row["single_forward_ms"] = round(_events(lambda: m(images), 1 if S > 96 else args.reps), 1)
                row["single_over_reconstruct"] = round(row["single_forward_ms"] / rec_ms, 2)
            except torch.cuda.OutOfMemoryError:
                row["single_forward_ms"] = "did not fit"
            torch.cuda.empty_cache()
        else:
            row["single_forward_ms"] = "not run"
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(dict(info, rows=rows)))


if __name__ == "__main__":
    main()
