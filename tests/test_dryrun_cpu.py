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
    assert dry.args("ovg_aggregator_forward")[0][1] is None and all(a[2] == 0 for a in dry.args("ovg_dpt_forward"))
    assert n("ovg_camera_create") == 1 and n("ovg_camera_forward") == 1
    c = dry.descs["ovg_camera_create"]
    assert (c.D, c.heads, c.trunk_depth) == (256, 2, 2) and c.trunk[1].w_fc2 and not c.trunk[0].qn_w and c.fc2_w and c.mod_w
    a = dry.descs["ovg_aggregator_create"]
    assert (a.C, a.registers, a.depth, a.patch) == (128, 4, 4, 14) and list(a.keep_layers) == [0, 1, 2, 3]
    assert a.frame_blocks[3].qn_w and a.global_blocks[0].w_qkv and a.depth_w and a.ones_c
    p = dry.descs["ovg_dpt_create"]
    assert (p.C2, p.feat, p.patch) == (256, 128, 14) and list(p.oc) == [64, 128, 256, 256] and p.outc in (2, 4)
    assert not p.fus[3].rcu1[0] and p.fus[0].rcu1[0] and p.fus[3].rcu2[3] and p.up_w[1] and p.down_w


def test_context_parallel_forward_runs_the_rank_views(dry):
    """Rank 1 of 2 on a 4-view scene: the aggregator, DINOv2 and DPT heads run over views 2..3, the depth normalisation sees
    every selected view of the scene, and the camera head reads the camera tokens of all 4 views."""
    import ctypes as C
    from omnivggt_official_b200 import _lib as L
    from omnivggt_official_b200.context_parallel import ContextParallel
    from omnivggt_official_b200.engine import Engine

    S = 4
    m = mini_model("mini_dino").eval()
    m.use_cuda_graph = False
    m._engine = Engine(m)

    class Stand(ContextParallel):            # no process group: the descriptor is filled, the camera tokens are a host tensor
        def __init__(self):
            self.rank, self.world = 1, 2
            self.cam_all = torch.zeros(S, 2 * m.embed_dim)

        def desc(self, heads, ntok_total, views_total):
            d = L.ContextParallelDesc()
            d.rank, d.world, d.views_total = self.rank, self.world, views_total
            return d

    m._cp = Stand()
    inp = make_inputs(1, S, 28, 28, seed=1)
    out = m(depth_gt_index=[0, 3], camera_gt_index=[1], **inp)

    def ints(p, n):
        return list((C.c_int * n).from_address(p)) if n else []

    assert dry.count("ovg_aggregator_forward") == 1
    a = dry.args("ovg_aggregator_forward")[0]
    assert a[1] is not None and a[13:15] == (1, 2) and a[21] is None        # cp, B = 1, S = 2, no layer export
    assert ints(a[6], a[7]) == [0, 3] and ints(a[8], a[9]) == [3]           # scene indices: all selected, this rank's
    assert dry.count("ovg_dino_forward") == 1 and dry.args("ovg_dino_forward")[0][5] == 2
    cam = dry.args("ovg_camera_forward")
    assert len(cam) == 1 and cam[0][1] == m._cp.cam_all.data_ptr() and cam[0][2:4] == (1, S)
    dpt = dry.args("ovg_dpt_forward")
    assert len(dpt) == 2 and all(d[2] == 0 and d[6] == 2 for d in dpt)     # bf16 slots, one chunk of the rank's 2 frames
    assert out["view_range"] == (2, 4) and torch.equal(out["images"], inp["images"][:, 2:4])
    assert out["depth"].shape == (1, 2, 28, 28, 1) and out["pose_enc"].shape == (1, S, 9)
