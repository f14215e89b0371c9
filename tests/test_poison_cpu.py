"""The poisoning allocator of test_poison_gpu.py (CPU): what it hands out, and that the package still allocates every
workspace and output of the dry-run entry points through it, so that none of them drops out of the poison test."""
import struct

import pytest
import torch

from oracle.synth import make_inputs
from ovg_support import dry_workspaces, mini_model, scene  # noqa: F401  (fixture "dry")
from test_poison_gpu import GUARD, GUARD_BYTE, PACKAGE_MODULES, poison  # noqa: F401  (fixture)


def _payload(P, t):
    raw, n, _ = next(a for a in P.allocs if a[0].data_ptr() + GUARD == t.data_ptr())
    return raw, n


def test_proxy_shapes_dtypes_poison_and_guards(poison):
    from omnivggt_official_b200 import engine, ops
    saved = {m: getattr(__import__(f"omnivggt_official_b200.{m}", fromlist=["torch"]), "torch") for m in PACKAGE_MODULES}
    f32_finite = struct.unpack("<f", bytes([0x3F] * 4))[0]
    for pattern, fval, ival in (("nan", None, -1), ("zero", 0.0, 0), ("finite", f32_finite, -1)):
        with poison(pattern, devices=("cpu",)) as P:
            assert engine.torch is P and ops.torch is P
            cases = [P.empty(3, 5, dtype=torch.float32, device="cpu"), P.empty((2, 7), dtype=torch.bfloat16, device="cpu"),
                     P.empty(torch.Size([4]), dtype=torch.float16, device="cpu"), P.empty((), dtype=torch.float32, device="cpu"),
                     P.empty(0, 3, dtype=torch.float32, device="cpu"), P.empty(9, dtype=torch.int64, device="cpu"),
                     P.empty(11, dtype=torch.int32, device="cpu"), P.empty(13, dtype=torch.uint8, device="cpu")]
            like = P.empty_like(cases[0])
            shapes = [(3, 5), (2, 7), (4,), (), (0, 3), (9,), (11,), (13,)]
            for t, s in zip(cases, shapes):
                assert tuple(t.shape) == s and t.is_contiguous()
            assert like.shape == (3, 5) and like.dtype == torch.float32
            for t in cases[:4] + [like]:                                        # (an empty tensor's data_ptr() is 0)
                raw, n = _payload(P, t)
                assert n == t.numel() * t.element_size() and t.data_ptr() % 16 == 0
                assert (raw[:GUARD] == GUARD_BYTE).all() and (raw[GUARD + n:] == GUARD_BYTE).all() and len(raw) == 2 * GUARD + n
                assert (raw[GUARD:GUARD + n] == {"nan": 0xFF, "zero": 0, "finite": 0x3F}[pattern]).all()
                assert torch.isnan(t.float()).all() if fval is None else torch.isfinite(t.float()).all()
            if pattern == "finite":
                assert cases[0][0, 0].item() == f32_finite and abs(f32_finite - 0.747) < 1e-3
            for t in cases[5:7]:
                assert (t == ival).all()
            assert (cases[7] == (255 if pattern != "zero" else 0)).all()      # never the finite pattern: indices stay 0 or -1
            z = P.zeros(5, device="cpu")
            assert (z == 0).all() and any(s <= z.data_ptr() < e for s, e in P.ranges())
            assert P.empty(3, dtype=torch.float32, device="cpu", pin_memory=False).shape == (3,)
            assert P.guards_broken() == []
            i = next(k for k, a in enumerate(P.allocs) if a[0].data_ptr() + GUARD == cases[6].data_ptr())
            raw, n, _ = P.allocs[i]
            raw[GUARD + n] = 0                                                  # one byte past the end
            assert P.guards_broken() == [i]
            raw[GUARD - 1] = 0                                                  # one byte before the start
            assert P.guards_broken() == [i]
    for m, t in saved.items():
        assert getattr(__import__(f"omnivggt_official_b200.{m}", fromlist=["torch"]), "torch") is t
    with poison("nan") as P:                                                    # CPU tensors are not poisoned by default
        t = P.empty(4, device="cpu")
        assert P.allocs == [] and t.shape == (4,)


# ovg_* entry point -> positions of its workspace and output pointers (a ctypes array: every element)
PTR_ARGS = {
    "ovg_aggregator_forward": (17, 19, 20, 21), # workspace, slots, cam_out, layers
    "ovg_dino_forward": (8, 10),                # workspace, patch tokens
    "ovg_dpt_forward": (13, 14, 15),            # preds, conf, workspace
    "ovg_camera_forward": (5, 6),               # out, workspace
    "ovg_conf_percentile_mask": (4, 5, 6, 7),   # workspace, mask, threshold, count
    "ovg_point_cloud_count": (7, 9),            # workspace, count
    "ovg_point_cloud_center": (2, 4),           # workspace, centre
}


def _pointers(name, args):
    out = []
    for i in PTR_ARGS[name]:
        v = args[i]
        vals = list(v) if hasattr(v, "_length_") else [v]
        out += [(i, p) for p in vals if p]
    return out


def _coverage(rec, P, want):
    ranges = P.ranges()
    seen = set()
    for name, args in rec.calls:
        if name.endswith(("_create", "_destroy", "_workspace_bytes")):
            continue
        assert name in PTR_ARGS, f"{name}: entry point without a workspace / output map in PTR_ARGS"
        seen.add(name)
        for i, p in _pointers(name, args):
            assert any(s <= p < e for s, e in ranges), f"{name} argument {i} was not allocated by the poisoning proxy"
    print("entry points checked:", sorted(seen))
    assert seen == want, seen ^ want


def test_dry_run_forward_allocates_every_pointer_through_the_proxy(dry, poison):
    """Forward of the DINOv2 variant with depth and camera aux and 9 views (DPT chunks of 8 and 1)."""
    from omnivggt_official_b200.engine import Engine
    m = mini_model("mini_dino").eval()
    with poison("nan", devices=("cpu",)) as P:
        m._engine = Engine(m)
        inp = make_inputs(1, 9, 28, 28, seed=1)
        out = m(depth_gt_index=[4], camera_gt_index=[0, 3], **inp)
        assert out["depth"].shape == (1, 9, 28, 28, 1)
        assert dry.count("ovg_dpt_forward") == 4
        assert {"agg_ws", "dino_ws", "cam.ws", "depth_head.ws", "point_head.ws"} <= set(m._engine.ws.bufs)
        _coverage(dry, P, {"ovg_aggregator_forward", "ovg_dino_forward", "ovg_dpt_forward", "ovg_camera_forward"})
        assert P.guards_broken() == []


def test_dry_run_point_cloud_allocates_through_the_proxy(dry, poison):
    from omnivggt_official_b200 import OmniVGGT
    with poison("nan", devices=("cpu",)) as P:
        OmniVGGT.point_cloud(scene(3, 6, 8, distinct_cameras=True), mask_black_bg=True)
        _coverage(dry, P, {"ovg_conf_percentile_mask", "ovg_point_cloud_count", "ovg_point_cloud_center"})
