"""Component calls and heads set to None (GPU).

  - model.aggregator / camera_head / depth_head / point_head compose to exactly what forward() returns (bit for bit, eager);
  - the exported fp32 layers against the reference's aggregated_tokens_list (goldens' agg_first / agg_last);
  - the reference's fp32 token list (CPU oracle) through these heads against the oracle's heads;
  - the kernels: ovg_dpt_forward_f32 on fp32 layers equals ovg_dpt_forward on their bf16 rounding, and the fp32 export writes
    the same values the bf16 snapshots and the camera tokens hold;
  - forward with heads set to None: the other outputs are unchanged, in eager and in CUDA-graph replay."""
import json
import os

import pytest
import torch
from safetensors.torch import load_file

from conftest import GOLDEN, golden_index, golden_schema
from oracle import omnivggt_oracle as O
from oracle.synth import make_inputs, make_state_dict
from test_model_gpu import build, rel

pytestmark = pytest.mark.gpu
INDEX = golden_index()
TOL = 2e-2
HEADS = ("camera_head", "depth_head", "point_head")
KEYS = ("pose_enc", "depth", "depth_conf", "world_points", "world_points_conf")


def _record(line):
    """Print a measured value; with OVG_TEST_RECORD set to a file path, also append it there."""
    print(line)
    path = os.environ.get("OVG_TEST_RECORD")
    if path:
        with open(path, "a") as f:
            f.write(line + "\n")


_MODELS = {}


def model(variant):
    if variant not in _MODELS:
        if variant == "full_width":
            from omnivggt_official_b200 import OmniVGGT
            m = OmniVGGT(img_size=518, depth=4, dino_depth=2, dpt_layers=(0, 1, 2, 3), camera_trunk_depth=2)
            m.load_state_dict(make_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, 0))
            _MODELS[variant] = m.cuda().eval()
        else:
            _MODELS[variant] = build(variant)
    m = _MODELS[variant]
    m.use_cuda_graph = False
    return m


def cuda_inputs(B, S, H, W, seed):
    return {k: v.cuda() for k, v in make_inputs(B, S, H, W, seed=seed).items()}


COMPOSE = {   # variant, B, S, H, W, depth_gt_index, camera_gt_index
    "images_only": ("mini_conv", 1, 3, 56, 56, [], []),
    "partial_aux_b2": ("mini_conv", 2, 4, 56, 56, [0, 2], [0, 1, 3]),
    "rect": ("mini_conv", 1, 2, 42, 70, [0, 1], [0, 1]),
    "chunked_s9": ("mini_conv", 1, 9, 42, 42, [3], [0, 5]),
    "dino_rect": ("mini_dino", 1, 2, 42, 70, [], [1]),
    "full_width": ("full_width", 1, 3, 154, 210, [0, 2], [0, 1]),
}


@pytest.mark.parametrize("case", sorted(COMPOSE))
def test_components_compose_to_forward_bit_for_bit(case):
    variant, B, S, H, W, didx, cidx = COMPOSE[case]
    m = model(variant)
    inp = cuda_inputs(B, S, H, W, seed=50 + B * S)
    out = m(**inp, depth_gt_index=didx, camera_gt_index=cidx)
    layers, ps = m.aggregator(**inp, depth_gt_index=didx, camera_gt_index=cidx)
    assert ps == 5 and len(layers) == len(m.aggregator.frame_blocks)
    poses = m.camera_head(layers)
    depth, depth_conf = m.depth_head(layers, inp["images"], ps)
    points, points_conf = m.point_head(layers, images=inp["images"], patch_start_idx=ps)
    torch.cuda.synchronize()
    assert len(poses) == len(out["pose_enc_list"]) == 4
    for a, b in zip(poses, out["pose_enc_list"]):
        assert torch.equal(a, b)
    for k, t in (("depth", depth), ("depth_conf", depth_conf), ("world_points", points), ("world_points_conf", points_conf)):
        assert t.shape == out[k].shape and torch.equal(t, out[k]), k


@pytest.mark.parametrize("case", ["conv_partial_aux_b2", "dino_rect_interp"])
def test_exported_layers_match_the_reference_tokens(case):
    meta = INDEX[case]
    m = model(meta["variant"])
    B, S, H, W = meta["B"], meta["S"], meta["H"], meta["W"]
    inp = cuda_inputs(B, S, H, W, seed=meta["input_seed"])
    layers, ps = m.aggregator(**inp, depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"])
    torch.cuda.synchronize()
    ref = load_file(os.path.join(GOLDEN, f"{case}.safetensors"))
    T = (H // 14) * (W // 14) + 5
    assert ps == 5 and len(layers) == 4
    for t in layers:
        assert t.shape == (B, S, T, 256) and t.dtype == torch.float32 and t.is_cuda and torch.isfinite(t).all()
    errs = {"agg_first": rel(layers[0], ref["agg_first"]), "agg_last": rel(layers[-1], ref["agg_last"])}
    _record(f"exported layers {case} " + json.dumps({k: round(v, 6) for k, v in errs.items()}))
    assert errs["agg_first"] < TOL and errs["agg_last"] < TOL, errs


def test_reference_tokens_into_these_heads():
    """The oracle's fp32 aggregated_tokens_list, computed on the CPU, through model.depth_head / point_head / camera_head,
    against the oracle's own heads on the same list."""
    meta = INDEX["conv_partial_aux_b2"]
    v = golden_schema("mini_conv")["variant"]
    sd = make_state_dict(golden_schema("mini_conv")["schema"], 0)
    m = model("mini_conv")
    B, S, H, W = meta["B"], meta["S"], meta["H"], meta["W"]
    inp = make_inputs(B, S, H, W, seed=meta["input_seed"])
    cfg = O.OracleConfig(dpt_layers=(0, 1, 2, 3), camera_head_heads=v["cam_heads"])
    inter, ns = O.aggregator(sd, inp["images"], inp["extrinsics"], inp["intrinsics"], inp["depth"], inp["mask"],
                             meta["depth_gt_index"], meta["camera_gt_index"], cfg)
    tokens = [inter[i] for i in range(len(inter))]
    want = {}
    want["depth"], want["depth_conf"] = O.dpt_head(sd, "depth_head", inter, H, W, ns, cfg, "exp")
    want["world_points"], want["world_points_conf"] = O.dpt_head(sd, "point_head", inter, H, W, ns, cfg, "inv_log")
    want_pose = O.camera_head(sd, "camera_head", inter[len(inter) - 1], cfg)
    gpu_tokens = [t.cuda() for t in tokens]
    images = inp["images"].cuda()
    got = {}
    got["depth"], got["depth_conf"] = m.depth_head(gpu_tokens, images, ns)
    got["world_points"], got["world_points_conf"] = m.point_head(gpu_tokens, images, ns)
    poses = m.camera_head(tokens)                                  # CPU tensors are moved to the device
    errs = {k: rel(got[k], want[k]) for k in want}
    for i in range(4):
        errs[f"pose_enc_list.{i}"] = rel(poses[i], want_pose[i])
    _record("oracle tokens into heads " + json.dumps({k: round(v, 6) for k, v in errs.items()}))
    for k, e in errs.items():
        assert e < TOL, (k, errs)


_FULL = {}


def full_heads_model(dpt_dtype):
    """The full-width DPT heads (C2 = 2048, features 256, out channels 256..1024) at 518 x 518, where the fused output tail runs."""
    if "m" not in _FULL:
        from omnivggt_official_b200 import OmniVGGT
        with torch.device("cuda"):
            m = OmniVGGT(depth=4, dino_depth=1, dpt_layers=(0, 1, 2, 3), camera_trunk_depth=1, init_seed=None)
        _FULL["m"] = m.randomize_(3).eval()
    m = _FULL["m"]
    if m.dpt_dtype != dpt_dtype:
        m.dpt_dtype = dpt_dtype
        m._invalidate()
    return m


@pytest.mark.parametrize("dpt_dtype", ["fp16", "bf16"])
@pytest.mark.parametrize("name,act", [("depth_head", 0), ("point_head", 1)])
def test_dpt_forward_f32_equals_bf16_slots(dpt_dtype, name, act):
    from omnivggt_official_b200 import _lib as L
    m = full_heads_model(dpt_dtype)
    eng = m.engine()
    K, H, W = 3, 518, 518
    assert L.lib().ovg_dpt_tail_supported(4 * 37 * 2, 4 * 37 * 2, H, W, 128) == 1        # the fused tail is on this path
    T = 37 * 37 + 5
    g = torch.Generator(device="cuda").manual_seed(7)
    x = {i: torch.randn(K, T, 2048, device="cuda", generator=g) * (1.0 + i) for i in m.dpt_layers}
    eng.warm_tables(H, W)
    a = eng.dpt(name, x, m.dpt_layers, K, H, W, head_act=act, out=eng.dpt_alloc(name, K, H, W))
    b = eng.dpt(name, {i: t.to(torch.bfloat16) for i, t in x.items()}, m.dpt_layers, K, H, W, head_act=act,
                out=eng.dpt_alloc(name, K, H, W))
    torch.cuda.synchronize()
    for u, w in zip(a, b):                                    # bit patterns: equal even where an activation overflowed
        assert torch.equal(u.view(torch.int32), w.view(torch.int32))
    _record(f"dpt f32 vs bf16 {name} {dpt_dtype}: finite fraction {torch.isfinite(a[0]).float().mean().item():.4f}")


@pytest.mark.parametrize("variant", ["mini_conv", "full_width"])
def test_layer_export_agrees_with_snapshots_and_camera_tokens(variant):
    """One ovg_aggregator_forward_layers call writing slots and layers: every kept slot is the bf16 rounding of its layer; the
    camera tokens are token 0 of the last layer; and ovg_aggregator_forward without layers writes the same slots and camera
    tokens bit for bit (the export does not perturb the forward)."""
    m = model(variant)
    eng = m.engine()
    B, S, H, W = (2, 3, 42, 70) if variant == "mini_conv" else (1, 3, 154, 210)
    didx, cidx = [1], [0, 2]
    inp = cuda_inputs(B, S, H, W, seed=61)
    args = (inp["images"], inp["extrinsics"], inp["intrinsics"], inp["depth"], inp["mask"], didx, cidx)
    slots, cam = m._aggregate(eng, *args)
    slots0 = {i: t.clone() for i, t in slots.items()}
    cam0 = cam.clone()
    T = (H // 14) * (W // 14) + 5
    layers = [torch.empty(B * S, T, 2 * eng.C, device="cuda") for _ in range(eng.depth)]
    slots, cam = m._aggregate(eng, *args, layers=layers)
    torch.cuda.synchronize()
    assert torch.equal(cam, cam0) and torch.equal(cam, layers[-1][:, 0])
    for i in m.dpt_layers:
        assert torch.equal(slots[i], slots0[i]), i
        assert torch.equal(slots[i], layers[i].to(torch.bfloat16)), i


VARIANTS = {"no_point": ("point_head",), "no_dpt": ("depth_head", "point_head"), "no_camera": ("camera_head",)}


@pytest.mark.parametrize("variant", ["mini_conv", "full_width"])
@pytest.mark.parametrize("drop", sorted(VARIANTS))
def test_none_heads_leave_the_other_outputs_unchanged(variant, drop):
    m = model(variant)
    B, S, H, W = (1, 3, 56, 56) if variant == "mini_conv" else (1, 2, 154, 210)
    inp = cuda_inputs(B, S, H, W, seed=71)
    kw = dict(depth_gt_index=[1], camera_gt_index=[0, 1])
    full = m(**inp, **kw)
    saved = {n: getattr(m, n) for n in VARIANTS[drop]}
    try:
        for n in saved:
            setattr(m, n, None)
        assert m._engine is None
        m.use_cuda_graph = True
        outs = [m(**inp, **kw) for _ in range(3)]                   # the third call is captured and replayed
        assert any(e["graph"] is not None for e in m._graphs.values()), "graph was not captured"
        gone = {k for n in saved for k in {"camera_head": ("pose_enc", "pose_enc_list"), "depth_head": ("depth", "depth_conf"),
                                           "point_head": ("world_points", "world_points_conf")}[n]}
        for out in (outs[0], outs[2]):
            assert set(out) == (set(full) - gone)
            for k in out:
                if k == "pose_enc_list":
                    assert all(torch.equal(a, b) for a, b in zip(out[k], full[k]))
                elif k != "images":
                    assert torch.equal(out[k], full[k]), k
    finally:
        for n, mod in saved.items():
            setattr(m, n, mod)
        m.use_cuda_graph = False
    again = m(**inp, **kw)
    assert set(again) == set(full)
    for k in KEYS:
        assert torch.equal(again[k], full[k]), k
