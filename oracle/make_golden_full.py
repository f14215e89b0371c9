"""Full-size parity pins: run the UNMODIFIED reference ``OmniVGGT`` (24 + 24 aggregator blocks, DINOv2 ViT-L patchifier,
camera head, both DPT heads; reference omnivggt/models/omnivggt.py:10-68) once per case at that case's image size on CPU fp32
and store its outputs (build container only; TEST INFRASTRUCTURE).

    python oracle/make_golden_full.py [case ...]   # all nine: ~12 min on 8 cores, peak host memory 17.2 GB (full_cfg5)

Cases (bench.CONFIGS / BASELINE.json configs):
  full_cfg1      cfg1: 1 scene x 4 views, images only
  full_aux_s3    cfg3-shaped: 1 scene x 3 views, depth + camera aux on every view
  full_mixed_s5  cfg5-shaped: 1 scene x 5 views, partial depth_gt_index / camera_gt_index
  full_cfg2      cfg2: 1 scene x 8 views, images only (the reference's DPT heads take all 8 frames in one chunk)
  full_cfg3      cfg3: 1 scene x 8 views, depth + camera aux on every view
  full_cfg5      cfg5: 1 scene x 24 views, the sparse index lists of bench.CONFIGS["cfg5"] (3 DPT chunks of 8 frames)
  full_land_s10  392 x 518 (a 4:3 photo): 10 views, depth aux on views 1 and 8, camera aux on 0 / 4 / 9 (DPT chunks 8 + 2)
  full_wide_s5   294 x 518 (a 16:9 frame): 5 views, images only; 21 patch rows, so the stride-2 level is 11 x 19
  full_tall_s3   882 x 518 (the tallest input the engine accepts): 3 views, depth + camera aux on every view; 63 patch rows
The first six are 518 x 518; the index lists of full_cfg2/3/5 are read from bench.CONFIGS so they cannot drift from what
bench.py runs.  The loaders fix the width at 518 and scale the height, so the last three are the shapes real photos produce.

Weights are oracle/synth.make_state_dict(schema, seed 0) over the reference's own 1 505-key schema (stored as
tests/golden/full.schema.json, names + shapes only), so the GPU tests rebuild the identical state dict without the
reference.  Dense outputs are stored at the row x column lists of oracle/full_golden.lines (recorded in full_index.json):
stride 7 from 3 for the first three cases, stride 13 from 6 for full_cfg2 / full_cfg3 and the non-square cases, and stride
15 from 7 for full_cfg5 (13 and 15 are coprime to the 14-pixel patch, so every position inside a patch is sampled on both
axes), each plus the two outermost lines per side.  Every fixture stays under 1 MB.
"""
from __future__ import annotations

import json
import os
import resource
import sys
import time

import torch
from safetensors.torch import save_file

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from bench import CONFIGS  # noqa: E402
from oracle.full_golden import GOLDEN, lines, sample  # noqa: E402
from oracle.ref_shims import import_reference  # noqa: E402
from oracle.synth import make_inputs, make_state_dict  # noqa: E402

SQUARE = (518, 518)


def _bench(cfg):
    c = CONFIGS[cfg]
    return c["S"], list(c["depth_idx"]), list(c["cam_idx"])


# name -> ((H, W), S, depth_gt_index, camera_gt_index, input seed, stride, offset)
CASES = {
    "full_cfg1": (SQUARE, 4, [], [], 11, 7, 3),
    "full_aux_s3": (SQUARE, 3, [0, 1, 2], [0, 1, 2], 12, 7, 3),
    "full_mixed_s5": (SQUARE, 5, [0, 3], [0, 2, 4], 13, 7, 3),
    "full_cfg2": (SQUARE, *_bench("cfg2"), 14, 13, 6),
    "full_cfg3": (SQUARE, *_bench("cfg3"), 15, 13, 6),
    "full_cfg5": (SQUARE, *_bench("cfg5"), 16, 15, 7),       # 24 views: the sparser stride keeps the fixture under 1 MB
    "full_land_s10": ((392, 518), 10, [1, 8], [0, 4, 9], 17, 13, 6),
    "full_wide_s5": ((294, 518), 5, [], [], 18, 13, 6),
    "full_tall_s3": ((882, 518), 3, [0, 1, 2], [0, 1, 2], 19, 13, 6),
}


def peak_rss_gb() -> float:
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20     # ru_maxrss is in KiB on Linux


def main():
    import_reference()
    from omnivggt.models.omnivggt import OmniVGGT as RefOmniVGGT
    torch.set_num_threads(os.cpu_count() or 8)
    only = set(sys.argv[1:]) or set(CASES)
    t0 = time.time()
    m = RefOmniVGGT().eval()
    schema = {k: list(t.shape) for k, t in m.state_dict().items()}
    sd = make_state_dict(schema, seed=0)
    m.load_state_dict(sd, strict=True)
    del sd
    with open(os.path.join(GOLDEN, "full.schema.json"), "w") as f:
        json.dump({"schema": schema}, f, indent=0, sort_keys=True)
    print(f"reference OmniVGGT built: {len(schema)} tensors, {time.time() - t0:.0f} s", flush=True)
    path = os.path.join(GOLDEN, "full_index.json")
    index = json.load(open(path)) if os.path.exists(path) else {}
    index = {k: v for k, v in index.items() if k in CASES}
    for name, ((H, W), S, didx, cidx, seed, stride, offset) in CASES.items():
        if name not in only:
            continue
        inp = make_inputs(1, S, H, W, seed=seed)
        t0 = time.time()
        with torch.no_grad():
            out = m(images=inp["images"], extrinsics=inp["extrinsics"], intrinsics=inp["intrinsics"], depth=inp["depth"],
                    mask=inp["mask"], depth_gt_index=list(didx), camera_gt_index=list(cidx))
        dt = time.time() - t0
        rows, cols = lines(H, stride, offset), lines(W, stride, offset)
        store = sample(out, rows, cols)
        save_file(store, os.path.join(GOLDEN, f"{name}.safetensors"))
        stats = {k: [float(v.abs().mean()), float(v.abs().max())] for k, v in store.items() if "list" not in k}
        index[name] = dict(S=S, H=H, W=W, depth_gt_index=didx, camera_gt_index=cidx, input_seed=seed, weight_seed=0,
                           stride=stride, offset=offset, rows=rows, cols=cols, cpu_forward_s=round(dt, 1), stats=stats)
        with open(path, "w") as f:        # after every case, so a long run leaves the finished cases usable
            json.dump(index, f, indent=1, sort_keys=True)
        print(name, f"{dt:.0f} s, peak host memory {peak_rss_gb():.1f} GB", stats, flush=True)
        del out, store


if __name__ == "__main__":
    main()
