"""Model-level parity (GPU): the drop-in OmniVGGT module (CUDA engine) against
  (a) golden outputs of the unmodified reference (tests/golden, reduced configs, all index patterns), and
  (b) the fp32 CPU oracle at full width (C = 1024, DINOv2 patchifier) on a reduced depth / image size,
plus size-independent properties at the BASELINE image size.

Tolerance.  The kernels compute with bf16 operands and fp32 accumulation (the reference runs fp32), so the bar is stated
as relative L2 per output: 2e-2 on the reduced configs / full-width model (measured: <= 1.5e-2, recorded in
DESIGN.md); pose_enc additionally max-abs 5e-2."""
import json
import os

import pytest
import torch
from safetensors.torch import load_file

from conftest import GOLDEN, golden_index, golden_schema
from oracle.synth import make_inputs, make_state_dict

pytestmark = pytest.mark.gpu
INDEX = golden_index()
TOL = 2e-2
TOL_FP16_HEADS = 1e-2        # full-size goldens with the default fp16 DPT heads (measured: <= 7.2e-3 on every output)
KEYS = ("pose_enc", "depth", "depth_conf", "world_points", "world_points_conf")


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def build(variant, dino_dtype=torch.float32):
    from omnivggt_official_b200 import OmniVGGT
    meta = golden_schema(variant)
    v = meta["variant"]
    kw = dict(img_size=v["img_size"], embed_dim=v["embed_dim"], depth=v["depth"], dpt_features=v["features"],
              dpt_out_channels=v["out_channels"], dpt_layers=tuple(range(v["depth"]))[-4:], camera_heads=v["cam_heads"],
              camera_trunk_depth=v["cam_trunk"], dino_dtype=dino_dtype)
    kw.update(patch_embed="conv") if v["patch_embed"] == "conv" else kw.update(patch_embed="dino", dino_depth=2, dino_heads=2)
    m = OmniVGGT(**kw)
    m.load_state_dict(make_state_dict(meta["schema"], 0), strict=True)
    return m.cuda().eval()


_MODELS = {}


def model(variant):
    if variant not in _MODELS:
        _MODELS[variant] = build(variant)
    return _MODELS[variant]


@pytest.mark.parametrize("case", sorted(INDEX))
def test_matches_reference_golden(case):
    meta = INDEX[case]
    m = model(meta["variant"])
    inp = {k: v.cuda() for k, v in make_inputs(meta["B"], meta["S"], meta["H"], meta["W"], seed=meta["input_seed"]).items()}
    out = m(depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"], **inp)
    torch.cuda.synchronize()
    ref = load_file(os.path.join(GOLDEN, f"{case}.safetensors"))
    errs = {k: rel(out[k], ref[k]) for k in KEYS}
    print(case, json.dumps(errs))
    d = os.path.join(os.path.dirname(GOLDEN), os.pardir, "gpurun_out")
    if os.path.isdir(d):
        with open(os.path.join(d, "model_parity_mini.txt"), "a") as f:
            f.write(case + " " + json.dumps({k: round(v, 5) for k, v in errs.items()}) + "\n")
    for k in KEYS:
        assert out[k].shape == ref[k].shape and out[k].dtype == torch.float32 and out[k].is_cuda
        assert torch.isfinite(out[k]).all(), k
        assert errs[k] < TOL, (k, errs)
    assert (out["pose_enc"].cpu() - ref["pose_enc"]).abs().max() < 5e-2
    assert len(out["pose_enc_list"]) == 4 and out["images"].shape == (meta["B"], meta["S"], 3, meta["H"], meta["W"])


def test_api_quirks_and_errors():
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 2, 56, 56, seed=11).items()}
    a = m(images=inp["images"][0])                           # 4-D input gets a batch dim (omnivggt.py:31-32)
    b = m(images=inp["images"], extrinsics=inp["extrinsics"], intrinsics=inp["intrinsics"], depth=torch.zeros_like(inp["depth"]),
          mask=torch.zeros_like(inp["mask"]), depth_gt_index=[], camera_gt_index=[])      # what inference.py passes
    assert torch.equal(a["depth"], b["depth"]) and a["images"].shape == (1, 2, 3, 56, 56)
    with pytest.raises(ValueError):
        m(images=torch.zeros(1, 2, 4, 56, 56, device="cuda"))
    with pytest.raises(AssertionError):
        m(images=torch.zeros(1, 2, 3, 50, 56, device="cuda"))


def test_batch_independence_and_determinism():
    """Scenes are independent (B is a pure batch dim): a scene's outputs do not depend on its batch neighbours, and a
    repeated call is bit-identical (no atomics on the path)."""
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(2, 3, 56, 56, seed=12).items()}
    both = m(depth_gt_index=[1], camera_gt_index=[0, 2], **inp)
    again = m(depth_gt_index=[1], camera_gt_index=[0, 2], **inp)
    one = m(depth_gt_index=[1], camera_gt_index=[0, 2], **{k: v[1:2] for k, v in inp.items()})
    for k in KEYS:
        assert torch.equal(both[k], again[k]), k
        assert rel(both[k][1:2], one[k]) < 2e-3, (k, rel(both[k][1:2], one[k]))


def test_cuda_graph_replay_matches_eager():
    """The third call of a signature is captured into a CUDA graph; replays must equal the eager launches bit for bit and
    must see new input values (static input buffers are refreshed)."""
    from omnivggt_official_b200 import OmniVGGT
    m = build("mini_conv")
    m.use_cuda_graph = True
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=31).items()}
    kw = dict(depth_gt_index=[1], camera_gt_index=[0, 2])
    eager = m(**inp, **kw)
    m(**inp, **kw)
    for _ in range(2):
        replay = m(**inp, **kw)
    key = next(iter(m._graphs))
    assert m._graphs[key]["graph"] is not None, "graph was not captured"
    for k in KEYS:
        assert torch.equal(eager[k], replay[k]), k
    inp2 = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=32).items()}
    r2 = m(**inp2, **kw)
    m.use_cuda_graph = False
    e2 = m(**inp2, **kw)
    for k in KEYS:
        assert torch.equal(r2[k], e2[k]), k
    assert not torch.equal(r2["depth"], replay["depth"])


def test_streaming_pipeline_matches_plain_forward():
    """pipeline.StreamingPipeline overlaps the H2D / D2H copies of neighbouring requests with the forward on separate streams;
    every request's pinned host result must equal the plain forward of the same inputs bit for bit, in graph replay too."""
    from omnivggt_official_b200.pipeline import StreamingPipeline
    m = build("mini_conv")
    m.use_cuda_graph = True
    kw = dict(depth_gt_index=[1], camera_gt_index=[0, 2])
    reqs = [{k: v.pin_memory() for k, v in make_inputs(1, 3, 56, 56, seed=40 + i).items()} for i in range(7)]
    want = [{k: v.cpu() for k, v in m(**{n: t.cuda() for n, t in r.items()}, **kw).items() if k in KEYS} for r in reqs]
    pipe = StreamingPipeline(m, slots=2, out_keys=KEYS)
    pending, got = [], []
    for r in reqs:
        pending.append(pipe.submit(r, **kw))
        if len(pending) > 1:
            got.append({k: v.clone() for k, v in pipe.result(pending.pop(0)).items()})
    got.append({k: v.clone() for k, v in pipe.result(pending.pop(0)).items()})
    pipe.drain()
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        for k in KEYS:
            assert torch.equal(g[k], w[k]), (i, k)


def test_view_permutation_equivariance():
    """Views 1..S-1 are exchangeable (no cross-frame position code; only view 0 uses the first camera/register slot)."""
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 4, 56, 56, seed=13).items()}
    perm = [0, 3, 1, 2]
    a = m(**inp, depth_gt_index=[], camera_gt_index=[])
    b = m(**{k: v[:, perm] for k, v in inp.items()}, depth_gt_index=[], camera_gt_index=[])
    for k in KEYS:
        assert rel(b[k], a[k][:, perm]) < 1e-2, (k, rel(b[k], a[k][:, perm]))


@pytest.mark.parametrize("aux", [False, True])
def test_full_width_vs_oracle(aux):
    """C = 1024 / 16 heads / DINOv2 ViT-L patchifier / DPT features 256 (the real widths) with depth 4 + 4 blocks and a
    154 x 210 image so that the fp32 CPU oracle finishes in seconds."""
    from omnivggt_official_b200 import OmniVGGT
    from oracle.omnivggt_oracle import OracleConfig, omnivggt_forward
    torch.manual_seed(0)
    m = OmniVGGT(img_size=518, depth=4, dino_depth=2, dpt_layers=(0, 1, 2, 3), camera_trunk_depth=2, dino_dtype=torch.float32)
    schema = {k: list(v.shape) for k, v in m.state_dict().items()}
    sd = make_state_dict(schema, 0)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    B, S, H, W = 1, 3, 154, 210
    inp = make_inputs(B, S, H, W, seed=21)
    didx, cidx = ([0, 2], [0, 1]) if aux else ([], [])
    out = m(depth_gt_index=didx, camera_gt_index=cidx, **{k: v.cuda() for k, v in inp.items()})
    torch.cuda.synchronize()
    ref = omnivggt_forward(sd, depth_gt_index=didx, camera_gt_index=cidx, cfg=OracleConfig(dpt_layers=(0, 1, 2, 3)), **inp)
    errs = {k: rel(out[k], ref[k]) for k in KEYS}
    print("full_width", aux, json.dumps(errs))
    for k in KEYS:
        assert errs[k] < TOL, errs


# ------------------------------------------------------------------------------------------- full-size parity pins
FULL_INDEX = json.load(open(os.path.join(GOLDEN, "full_index.json")))
_FULL = {}


def full_model():
    """The full architecture (24 + 24 blocks, DINOv2 ViT-L patchifier, 1 505 tensors) with the de-zeroed seed-0 weights the
    reference goldens were generated with (tests/golden/full.schema.json + oracle/synth.make_state_dict)."""
    if "m" not in _FULL:
        from omnivggt_official_b200 import OmniVGGT
        schema = json.load(open(os.path.join(GOLDEN, "full.schema.json")))["schema"]
        with torch.device("cuda"):
            m = OmniVGGT(init_seed=None)
        sd = make_state_dict(schema, 0)
        m.load_state_dict(sd, strict=True)       # same 1 505 keys as the reference module
        del sd
        _FULL["m"] = m.eval()
    return _FULL["m"]


@pytest.mark.parametrize("case,dpt_dtype", [(c, "fp16") for c in sorted(FULL_INDEX)] + [("full_cfg1", "bf16")])
def test_full_size_matches_reference_golden(case, dpt_dtype):
    """BASELINE.json configs[0] ("4 views @ 518 x 518 ... value check") and aux-shaped siblings: the full model on the CUDA
    path against outputs of the UNMODIFIED reference forward (omnivggt/models/omnivggt.py:20-68, CPU fp32; generated by
    oracle/make_golden_full.py).  Dense outputs are compared on the stored pixel lattice (every 7th row / column)."""
    meta = FULL_INDEX[case]
    m = full_model()
    if m.dpt_dtype != dpt_dtype:          # the heads' 16-bit format is fixed when the engine packs the weights
        m.dpt_dtype = dpt_dtype
        m._invalidate()
    st, o = meta["stride"], meta["stride"] // 2
    inp = {k: v.cuda() for k, v in make_inputs(1, meta["S"], meta["H"], meta["W"], seed=meta["input_seed"]).items()}
    out = m(depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"], **inp)
    torch.cuda.synchronize()
    ref = load_file(os.path.join(GOLDEN, f"{case}.safetensors"))
    got = {"pose_enc": out["pose_enc"]}
    for k in KEYS[1:]:
        assert torch.isfinite(out[k]).all(), k
        got[k] = out[k][:, :, o::st, o::st]
    errs = {k: rel(got[k], ref[k]) for k in KEYS}
    errs["pose_enc_maxabs"] = (out["pose_enc"].cpu() - ref["pose_enc"]).abs().max().item()
    for i in range(4):
        errs[f"pose_enc_list.{i}"] = rel(out["pose_enc_list"][i], ref[f"pose_enc_list.{i}"])
    line = f"{case} heads={dpt_dtype} S={meta['S']} depth_idx={meta['depth_gt_index']} cam_idx={meta['camera_gt_index']} " + json.dumps(
        {k: round(v, 5) for k, v in errs.items()})
    print(line)
    d = os.path.join(os.path.dirname(GOLDEN), os.pardir, "gpurun_out")
    if os.path.isdir(d):
        with open(os.path.join(d, "model_parity_full.txt"), "a") as f:
            f.write(line + "\n")
    for k in KEYS:
        assert got[k].shape == ref[k].shape, k
        assert errs[k] < (TOL if dpt_dtype == "bf16" else TOL_FP16_HEADS), (k, errs)


@pytest.mark.parametrize("S,didx,cidx", [(8, list(range(8)), list(range(8))),          # BASELINE.json configs[2]
                                         (24, [0, 3, 4, 11, 23], [0, 1, 7, 12, 20, 22])])  # configs[4]: 24 views, partial aux
def test_full_size_configs_properties(S, didx, cidx):
    """The full architecture (1 217.5 M parameters, 24 + 24 blocks, DINOv2 ViT-L patchifier) at 518 x 518 on the aux
    configurations BASELINE.json names.  The fp32 CPU oracle needs minutes at this size, so the checks are the
    size-independent ones: output contract, finiteness, run-to-run bit-determinism (eager and CUDA-graph replay agree),
    and that the auxiliary inputs of a view actually reach the predictions."""
    from omnivggt_official_b200 import OmniVGGT
    H = W = 518
    with torch.device("cuda"):
        m = OmniVGGT(init_seed=None)
    m.randomize_(0).eval()
    inp = {k: v.cuda() for k, v in make_inputs(1, S, H, W, seed=5).items()}
    outs = [m(depth_gt_index=didx, camera_gt_index=cidx, **inp) for _ in range(4)]   # call 3 captures, call 4 replays
    torch.cuda.synchronize()
    a = outs[0]
    assert a["depth"].shape == (1, S, H, W, 1) and a["world_points"].shape == (1, S, H, W, 3)
    assert a["depth_conf"].shape == (1, S, H, W) and a["pose_enc"].shape == (1, S, 9) and len(a["pose_enc_list"]) == 4
    for k in KEYS:
        assert torch.isfinite(a[k]).all(), k
        for o in outs[1:]:
            assert torch.equal(o[k], a[k]), k
    assert (a["depth"] > 0).all() and (a["depth_conf"] >= 1).all() and (a["world_points_conf"] >= 1).all()
    b = m(depth_gt_index=[], camera_gt_index=[], **inp)
    assert rel(b["depth"], a["depth"]) > 1e-4 and rel(b["pose_enc"], a["pose_enc"]) > 1e-4
    del m
    torch.cuda.empty_cache()
