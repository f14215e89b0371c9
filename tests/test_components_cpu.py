"""Component calls and heads set to None (CPU): the module against a recorder in place of the C library, as in
test_dryrun_cpu.py, looking at every call's arguments.  What is checked: which heads get a libovg handle, which entry points a
forward or a component call issues and with which pointers, the output keys for every subset of heads (reference
models/omnivggt.py:46-62), and that the owner back-references leave the parameter / state-dict / module tree unchanged."""
import copy
import itertools
import pickle

import pytest
import torch

from conftest import golden_schema
from oracle.synth import make_inputs
from ovg_support import dry, mini_model  # noqa: F401  (fixture)

HEADS = ("camera_head", "depth_head", "point_head")
KEYS = {"camera_head": ("pose_enc", "pose_enc_list"), "depth_head": ("depth", "depth_conf"),
        "point_head": ("world_points", "world_points_conf")}


def _model(variant="mini_conv"):
    m = mini_model(variant).eval()
    m.use_cuda_graph = False
    return m


def ready(m):
    """The engine of a CPU-resident model (OmniVGGT.engine() refuses a CPU model; the recorder stands in for the library)."""
    from omnivggt_official_b200.engine import Engine
    if m._engine is None:
        m._engine = Engine(m)
    return m._engine


def test_engine_creates_no_dpt_handle_for_a_none_head(dry):
    m = _model()
    m.point_head = None
    eng = ready(m)
    assert set(eng.dpt_packs) == {"depth_head"} and set(eng.h_dpt) == {"depth_head"}
    assert dry.count("ovg_dpt_create") == 1 and dry.count("ovg_camera_create") == 1


def test_pose_only_forward_writes_no_slot_exports_no_layer_and_runs_no_dpt(dry):
    m = _model()
    m.depth_head = None
    m.point_head = None
    ready(m)
    out = m(**make_inputs(1, 3, 56, 56, seed=1), depth_gt_index=[1], camera_gt_index=[0])
    assert set(out) == {"pose_enc", "pose_enc_list", "images"} and out["pose_enc"].shape == (1, 3, 9)
    assert dry.count("ovg_aggregator_forward") == 1
    args = dry.args("ovg_aggregator_forward")[0]
    assert args[1] is None and args[21] is None                             # one GPU, no layer export
    slots = args[19]
    assert len(slots) == 4 and all(p is None for p in slots)
    assert dry.count("ovg_dpt_create") == 0 and dry.count("ovg_dpt_forward") == 0 and dry.count("ovg_camera_forward") == 1
    assert not any(k.startswith("slot") for k in m._engine.ws.bufs)


@pytest.mark.parametrize("present", list(itertools.product([True, False], repeat=3)))
def test_output_keys_and_library_calls_follow_the_reference_gating(dry, present):
    m = _model()
    for name, on in zip(HEADS, present):
        if not on:
            setattr(m, name, None)
    ready(m)
    B, S, H, W = 2, 3, 42, 70
    out = m(**make_inputs(B, S, H, W, seed=2), depth_gt_index=[0], camera_gt_index=[0, 2])
    want = {"images"} | {k for name, on in zip(HEADS, present) if on for k in KEYS[name]}
    assert set(out) == want
    assert out["images"].shape == (B, S, 3, H, W)
    n_dpt = sum(present[1:])
    assert dry.count("ovg_dpt_create") == n_dpt and dry.count("ovg_dpt_forward") == n_dpt
    assert all(a[2] == 0 for a in dry.args("ovg_dpt_forward"))             # bf16 slots
    assert dry.count("ovg_camera_forward") == int(present[0])
    slots = dry.args("ovg_aggregator_forward")[0][19]
    assert all(p is None for p in slots) == (n_dpt == 0)
    if present[1]:
        assert out["depth"].shape == (B, S, H, W, 1) and out["depth_conf"].shape == (B, S, H, W)
    if present[2]:
        assert out["world_points"].shape == (B, S, H, W, 3)


def test_setting_a_head_invalidates_the_engine(dry):
    m = _model()
    eng = ready(m)
    m._graphs[("sig",)] = {"calls": 1, "graph": None}
    m.point_head = None
    assert m._engine is None and m._graphs == {}
    assert "point_head" not in ready(m).dpt_packs
    head = mini_model().point_head
    m.point_head = head
    assert m._engine is None and head.owner() is m
    assert "point_head" in ready(m).dpt_packs and eng is not m._engine


def test_aggregator_component_exports_every_layer_in_one_forward_call(dry):
    m = _model()
    ready(m)
    B, S, H, W = 2, 3, 42, 70
    layers, ps = m.aggregator(**make_inputs(B, S, H, W, seed=3), depth_gt_index=[1], camera_gt_index=[0])
    C2, depth = 2 * m.embed_dim, len(m.aggregator.frame_blocks)
    T = (H // 14) * (W // 14) + 5
    assert ps == 5 and len(layers) == depth
    assert all(t.shape == (B, S, T, C2) and t.dtype == torch.float32 for t in layers)
    assert dry.count("ovg_aggregator_forward") == 1
    args = dry.args("ovg_aggregator_forward")[0]
    assert args[1] is None                                                  # one GPU
    assert all(p is None for p in args[19])                                 # no bf16 slot: no DPT head reads them
    assert len(args[21]) == depth and list(args[21]) == [t.data_ptr() for t in layers]
    assert dry.count("ovg_dpt_forward") == 0 and dry.count("ovg_camera_forward") == 0


def test_head_components_pass_fp32_slots(dry):
    m = _model()
    ready(m)
    B, S, H, W = 1, 9, 28, 42
    T = (H // 14) * (W // 14) + 5
    tokens = [torch.zeros(B, S, T, 2 * m.embed_dim) for _ in range(4)]
    images = torch.zeros(B, S, 3, H, W)
    d, dc = m.depth_head(tokens, images, 5)
    p, pc = m.point_head(tokens, images=images, patch_start_idx=5, frames_chunk_size=4)
    assert d.shape == (B, S, H, W, 1) and dc.shape == (B, S, H, W) and p.shape == (B, S, H, W, 3) and pc.shape == (B, S, H, W)
    dpt = dry.args("ovg_dpt_forward")
    assert len(dpt) == 2 + 3 and all(a[2] == 1 for a in dpt)               # fp32 slots; chunks of 8, then of 4
    assert list(dpt[0][1]) == [t.data_ptr() for t in tokens] and dpt[0][3:5] == (T, 5)
    poses = m.camera_head(tokens, num_iterations=3)
    assert len(poses) == 3 and poses[0].shape == (B, S, 9)
    ct = dry.args("ovg_camera_forward")[0]
    assert ct[2:5] == (B, S, 3)
    with pytest.raises(ValueError):
        m.depth_head(tokens, torch.zeros(B, S, 3, 42, 42), 5)              # tokens do not match the image size


def test_component_calls_refuse_context_parallelism_and_detached_heads(dry):
    m = _model()
    head = m.depth_head
    m.depth_head = None
    ready(m)
    tokens = [torch.zeros(1, 2, 21, 256) for _ in range(4)]
    with pytest.raises(RuntimeError):
        head(tokens, torch.zeros(1, 2, 3, 56, 56), 5)
    m._cp = object()
    with pytest.raises(RuntimeError):
        m.aggregator(torch.zeros(1, 2, 3, 56, 56))
    with pytest.raises(RuntimeError):
        m.camera_head(tokens)


@pytest.mark.parametrize("variant", ["mini_conv", "mini_dino"])
def test_owner_references_leave_state_dict_and_modules_unchanged(variant):
    m = mini_model(variant)
    schema = golden_schema(variant)["schema"]
    assert set(m.state_dict()) == set(schema)
    assert set(m._modules) == {"aggregator", "camera_head", "point_head", "depth_head"}
    n_params = len(list(m.parameters()))
    n_modules = len(list(m.modules()))
    for name in ("aggregator", "camera_head", "depth_head", "point_head"):
        sub = getattr(m, name)
        assert sub.owner() is m and "_owner" not in sub._modules and "_owner" not in sub._parameters
    assert len(list(m.parameters())) == n_params and len(list(m.modules())) == n_modules
    c = copy.deepcopy(m)
    assert c.depth_head.owner() is c and m.depth_head.owner() is m
    r = pickle.loads(pickle.dumps(m))
    assert r.aggregator.owner() is r and set(r.state_dict()) == set(schema)
