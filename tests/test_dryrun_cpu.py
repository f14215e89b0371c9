"""Host-logic dry run (CPU): the boundary module + engine against a recorder in place of the C library.  The launch
SEQUENCES live in C++ (csrc/runtime.inc) and are covered by the -m gpu goldens; what is checked here is the Python side of the
runtime API: one handle per component, one forward call per component and DPT chunk, descriptors filled from the packed
weights, shapes of the returned dict -- for every aux / chunking / shape path."""
import pytest
import torch

from oracle.synth import make_inputs
from ovg_support import dry_workspaces, mini_model  # noqa: F401  (fixture "dry")


def test_runtime_calls_dino_backend(dry):
    from omnivggt_official_b200.engine import Engine
    m = mini_model("mini_dino").eval()
    m._engine = Engine(m)
    assert m._engine.dino is not None
    inp = make_inputs(1, 2, 42, 70, seed=1)
    out = m(images=inp["images"])
    assert out["depth"].shape == (1, 2, 42, 70, 1)
    n = dry.count
    assert n("ovg_dino_create") == 1 and n("ovg_dino_forward") == 1 and n("ovg_aggregator_forward") == 1
    d = dry.descs["ovg_dino_create"]
    assert (d.C, d.registers, d.depth, d.patch, d.kpad) == (128, 4, 2, 14, 592) and d.blocks[1].w_fc2 and not d.blocks[0].qn_w


@pytest.mark.parametrize("B,S,H,W,didx,cidx", [(1, 2, 56, 56, [], []), (2, 3, 42, 70, [0, 2], [0, 1]), (1, 9, 28, 28, [4], [0])])
def test_runtime_calls(dry, B, S, H, W, didx, cidx):
    from omnivggt_official_b200.engine import Engine
    m = mini_model().eval()
    m._engine = Engine(m)
    inp = make_inputs(B, S, H, W, seed=1)
    out = m(depth_gt_index=didx, camera_gt_index=cidx, **inp)
    assert out["depth"].shape == (B, S, H, W, 1) and out["world_points"].shape == (B, S, H, W, 3)
    assert out["depth_conf"].shape == (B, S, H, W) and out["pose_enc"].shape == (B, S, 9)
    n = dry.count
    assert n("ovg_aggregator_create") == 1 and n("ovg_dpt_create") == 2 and n("ovg_dino_create") == 0
    assert n("ovg_aggregator_forward") == 1 and n("ovg_dpt_forward") == 2 * -(-B * S // 8)      # chunks of 8 frames per head
    assert n("ovg_camera_create") == 1 and n("ovg_camera_forward") == 1
    c = dry.descs["ovg_camera_create"]
    assert (c.D, c.heads, c.trunk_depth) == (256, 2, 2) and c.trunk[1].w_fc2 and not c.trunk[0].qn_w and c.fc2_w and c.mod_w
    a = dry.descs["ovg_aggregator_create"]
    assert (a.C, a.registers, a.depth, a.patch) == (128, 4, 4, 14) and list(a.keep_layers) == [0, 1, 2, 3]
    assert a.frame_blocks[3].qn_w and a.global_blocks[0].w_qkv and a.depth_w and a.ones_c
    p = dry.descs["ovg_dpt_create"]
    assert (p.C2, p.feat, p.patch) == (256, 128, 14) and list(p.oc) == [64, 128, 256, 256] and p.outc in (2, 4)
    assert not p.fus[3].rcu1[0] and p.fus[0].rcu1[0] and p.fus[3].rcu2[3] and p.up_w[1] and p.down_w
