"""Workspace contract of every libovg entry point that carves a caller's workspace: a null workspace, a misaligned one and one a
byte shorter than the call needs are each refused with OVG_E_INVALID before any launch.  The call needs what its size query
answers, except where noted in cases().  The argument combinations in MISUSE are refused the same way with a well-formed
workspace.

The operands are placeholder device pointers, so the calls run in a child process that sees no CUDA device: an entry point
that wrongly accepted a workspace would fail with a CUDA error there instead of launching."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
OVG_E_INVALID = -1
PTR = 1 << 40                 # placeholder device pointer, aligned for every operand
V, CAP, NP = 3, 64, 2         # matches and tracks: views, points per view (H x W = 8 x 8), pairs
F, H, W = 2, 8, 8             # point cloud, mesh, sky, TSDF bounds
NX = 20                       # TSDF volume: NX^3 voxels


def placeholders(n):
    """A host array of n placeholder device pointers (the entry points read such arrays on the host)."""
    return (C.c_void_p * n)(*([PTR] * n))


def placeholder(t, v):
    """v of ctypes type t with every pointer in it, in nested arrays and structures too, set to PTR; other values kept."""
    if t is C.c_void_p:
        return PTR
    if issubclass(t, C.Array):
        return t(*(placeholder(t._type_, x) for x in v))
    if issubclass(t, C.Structure):
        for name, ft in t._fields_:
            setattr(v, name, placeholder(ft, getattr(v, name)))
    return v


def fill(desc, **ints):
    """desc with every pointer a placeholder and the given integer fields (or arrays of them) set."""
    placeholder(type(desc), desc)
    for name, value in ints.items():
        field = getattr(desc, name)
        setattr(desc, name, type(field)(*value) if isinstance(field, C.Array) else value)
    return desc


def handles(lib, L):
    """Runtime handles on placeholder weights: the aggregator, DINOv2, DPT and camera head.  Creating them makes no device call."""
    blocks = (L.BlockWeights * 1)(fill(L.BlockWeights()))
    out = {}
    for kind, desc in (
            ("aggregator", fill(L.AggregatorDesc(), C=64, registers=4, depth=1, patch=14, keep_layers=[0, 0, 0, 0])),
            ("dino", fill(L.DinoDesc(), C=64, registers=4, depth=1, patch=14, kpad=592)),
            ("dpt", fill(L.DptDesc(), C2=128, feat=64, patch=14, outc=4, oc=[64, 64, 64, 64], f16=0)),
            ("camera", fill(L.CameraDesc(), D=128, heads=2, trunk_depth=1))):
        for name, t in desc._fields_:
            if t is C.POINTER(L.BlockWeights):
                setattr(desc, name, blocks)
        h = C.c_void_p()
        L.check(getattr(lib, f"ovg_{kind}_create")(C.byref(desc), C.byref(h)))
        out[kind] = h
    return out


def cases(lib, L):
    """{entry point: (call(workspace, workspace_bytes), bytes the call needs, required alignment)}.  Tracks take a match
    workspace too: "<entry>(match)" breaks that one and keeps the tracks workspace well-formed."""
    hs = handles(lib, L)
    cp = fill(L.ContextParallelDesc(), rank=0, world=1, views_total=2)
    mean3 = (C.c_float * 3)(0.5, 0.5, 0.5)
    slots4, slots1 = placeholders(4), placeholders(1)
    n_cloud = F * H * W
    match_need = lib.ovg_match_workspace_bytes(V, CAP, NP)
    tracks_need = lib.ovg_tracks_workspace_bytes(V, CAP)

    def tracks_assign(mws, mwsb, ws, wsb):
        return lib.ovg_tracks_assign(PTR, PTR, NP, V, CAP, 1, mws, mwsb, ws, wsb, PTR, None)

    def tracks_gather(mws, mwsb, ws, wsb):
        return lib.ovg_tracks_gather(PTR, PTR, PTR, V, CAP, NP, W, 1, 2, mws, mwsb, ws, wsb, *([PTR] * 10), None)

    return {
        "ovg_point_cloud_count": (lambda ws, n: lib.ovg_point_cloud_count(PTR, PTR, F, H, W, 0, 0, ws, n, PTR, None),
                                  lib.ovg_point_cloud_workspace_bytes(n_cloud), 16),
        "ovg_point_cloud_gather": (lambda ws, n: lib.ovg_point_cloud_gather(PTR, PTR, PTR, F, H, W, 0, 0, 0, ws, n, PTR, PTR, PTR,
                                                                            PTR, n_cloud, None),
                                   lib.ovg_point_cloud_workspace_bytes(n_cloud), 16),
        "ovg_point_cloud_center": (lambda ws, n: lib.ovg_point_cloud_center(PTR, n_cloud, ws, n, PTR, None),
                                   lib.ovg_point_cloud_workspace_bytes(n_cloud), 16),
        # the scale uses the fixed-size head of the workspace only: the layout of one point
        "ovg_point_cloud_scale": (lambda ws, n: lib.ovg_point_cloud_scale(PTR, 100, 100, ws, n, PTR, None),
                                  lib.ovg_point_cloud_workspace_bytes(1), 16),
        "ovg_match_index": (lambda ws, n: lib.ovg_match_index(PTR, PTR, V, CAP, NP, ws, n, None), match_need, 256),
        "ovg_match_query": (lambda ws, n: lib.ovg_match_query(PTR, NP, V, CAP, ws, n, PTR, None), match_need, 256),
        "ovg_match_gather": (lambda ws, n: lib.ovg_match_gather(PTR, NP, V, CAP, W, ws, n, PTR, PTR, None), match_need, 256),
        "ovg_match_pair": (lambda ws, n: lib.ovg_match_pair(PTR, NP, V, CAP, 0, ws, n, PTR, PTR, None), match_need, 256),
        "ovg_tracks_assign": (lambda ws, n: tracks_assign(PTR, match_need, ws, n), tracks_need, 256),
        "ovg_tracks_assign(match)": (lambda ws, n: tracks_assign(ws, n, PTR, tracks_need), match_need, 256),
        "ovg_tracks_gather": (lambda ws, n: tracks_gather(PTR, match_need, ws, n), tracks_need, 256),
        "ovg_tracks_gather(match)": (lambda ws, n: tracks_gather(ws, n, PTR, tracks_need), match_need, 256),
        "ovg_bundle_adjust": (lambda ws, n: lib.ovg_bundle_adjust(PTR, PTR, PTR, PTR, PTR, PTR, 3, 10, 30, 5, 1, 0, 1.0, ws, n,
                                                                  *([PTR] * 7), None),
                              lib.ovg_ba_workspace_bytes(3, 10, 30), 256),
        "ovg_mesh_count": (lambda ws, n: lib.ovg_mesh_count(PTR, PTR, F, H, W, 0, 0, ws, n, PTR, None),
                           lib.ovg_mesh_workspace_bytes(F, H, W), 256),
        "ovg_mesh_faces": (lambda ws, n: lib.ovg_mesh_faces(PTR, None, 0, F, H, W, ws, n, PTR, PTR, None),
                           lib.ovg_mesh_workspace_bytes(F, H, W), 256),
        "ovg_mesh_compact": (lambda ws, n: lib.ovg_mesh_compact(PTR, PTR, F, H, W, ws, n, PTR, PTR, PTR, None),
                             lib.ovg_mesh_workspace_bytes(F, H, W), 256),
        # each TSDF call needs its own part of the workspace only
        "ovg_tsdf_bounds": (lambda ws, n: lib.ovg_tsdf_bounds(PTR, PTR, F, H, W, ws, n, PTR, None),
                            lib.ovg_tsdf_workspace_bytes(0, 0, 0, F, H, W), 256),
        "ovg_tsdf_integrate": (lambda ws, n: lib.ovg_tsdf_integrate(PTR, PTR, PTR, PTR, PTR, F, H, W, NX, NX, NX, 0.0, 0.0, 0.0,
                                                                    0.1, 0.4, ws, n, PTR, PTR, None),
                               lib.ovg_tsdf_workspace_bytes(NX, NX, NX, 0, 0, 0), 256),
        "ovg_tsdf_count": (lambda ws, n: lib.ovg_tsdf_count(PTR, NX, NX, NX, ws, n, PTR, None),
                           lib.ovg_tsdf_workspace_bytes(NX, NX, NX, 0, 0, 0), 256),
        "ovg_tsdf_extract": (lambda ws, n: lib.ovg_tsdf_extract(PTR, PTR, NX, NX, NX, 0.0, 0.0, 0.0, 0.1, ws, n, PTR, PTR, PTR,
                                                                None),
                             lib.ovg_tsdf_workspace_bytes(NX, NX, NX, 0, 0, 0), 256),
        "ovg_segment_sky": (lambda ws, n: lib.ovg_segment_sky(PTR, 1, 3 * H * W, 3, 1, F, H, W, None, ws, n, PTR, None, None),
                            lib.ovg_sky_workspace_bytes(F, H, W), 256),
        "ovg_farthest_point_sample": (lambda ws, n: lib.ovg_farthest_point_sample(PTR, 2, 5000, 16, None, 1, ws, n, PTR, None),
                                      lib.ovg_fps_workspace_bytes(2, 5000), 256),
        "ovg_compute_ranking": (lambda ws, n: lib.ovg_compute_ranking(PTR, 0, 10, 16, 4, 1, 1.0, 1, 0, 10, ws, n, PTR, PTR, None),
                                lib.ovg_ranking_workspace_bytes(10, 0), 256),
        "ovg_sim3_estimate": (lambda ws, n: lib.ovg_sim3_estimate(PTR, PTR, None, 100, ws, n, PTR, PTR, None),
                              lib.ovg_sim3_workspace_bytes(100), 256),
        "ovg_aggregator_forward": (
            lambda ws, n: lib.ovg_aggregator_forward(hs["aggregator"], None, PTR, PTR, None, None, None, 0, None, 0, PTR, PTR, 64, 1,
                                                     2, 28, 28, ws, n, slots4, PTR, None, None),
            lib.ovg_aggregator_workspace_bytes(hs["aggregator"], 1, 2, 28, 28, 0), 256),
        "ovg_aggregator_forward(layers)": (
            lambda ws, n: lib.ovg_aggregator_forward(hs["aggregator"], None, PTR, PTR, None, None, None, 0, None, 0, PTR, PTR, 64, 1,
                                                     2, 28, 28, ws, n, slots4, PTR, slots1, None),
            lib.ovg_aggregator_workspace_bytes(hs["aggregator"], 1, 2, 28, 28, 0), 256),
        "ovg_aggregator_forward(cp)": (
            lambda ws, n: lib.ovg_aggregator_forward(hs["aggregator"], C.byref(cp), PTR, PTR, None, None, None, 0, None, 0, PTR,
                                                     PTR, 64, 1, 2, 28, 28, ws, n, slots4, PTR, None, None),
            lib.ovg_aggregator_workspace_bytes(hs["aggregator"], 1, 2, 28, 28, 0), 256),
        # refused whatever the workspace: MISUSE
        "ovg_aggregator_forward(cp, layers)": (
            lambda ws, n: lib.ovg_aggregator_forward(hs["aggregator"], C.byref(cp), PTR, PTR, None, None, None, 0, None, 0, PTR,
                                                     PTR, 64, 1, 2, 28, 28, ws, n, slots4, PTR, slots1, None),
            lib.ovg_aggregator_workspace_bytes(hs["aggregator"], 1, 2, 28, 28, 0), 256),
        "ovg_aggregator_forward(depth_idx_local, no cp)": (
            lambda ws, n: lib.ovg_aggregator_forward(hs["aggregator"], None, PTR, PTR, PTR, PTR, PTR, 1, PTR, 1, PTR, PTR, 64, 1, 2,
                                                     28, 28, ws, n, slots4, PTR, None, None),
            lib.ovg_aggregator_workspace_bytes(hs["aggregator"], 1, 2, 28, 28, 1), 256),
        "ovg_dino_forward": (lambda ws, n: lib.ovg_dino_forward(hs["dino"], PTR, PTR, mean3, mean3, 2, 28, 28, ws, n, PTR, None),
                             lib.ovg_dino_workspace_bytes(hs["dino"], 2, 28, 28), 256),
        "ovg_dpt_forward": (lambda ws, n: lib.ovg_dpt_forward(hs["dpt"], slots4, 0, 9, 5, 0, 2, 28, 28, slots4, PTR, PTR, 0, PTR,
                                                              PTR, ws, n, None),
                            lib.ovg_dpt_workspace_bytes(hs["dpt"], 2, 28, 28), 256),
        "ovg_dpt_forward(f32)": (lambda ws, n: lib.ovg_dpt_forward(hs["dpt"], slots4, 1, 9, 5, 0, 2, 28, 28, slots4, PTR, PTR, 0,
                                                                   PTR, PTR, ws, n, None),
                                 lib.ovg_dpt_workspace_bytes(hs["dpt"], 2, 28, 28), 256),
        "ovg_dpt_forward(slots_f32 = 2)": (lambda ws, n: lib.ovg_dpt_forward(hs["dpt"], slots4, 2, 9, 5, 0, 2, 28, 28, slots4, PTR,
                                                                             PTR, 0, PTR, PTR, ws, n, None),
                                           lib.ovg_dpt_workspace_bytes(hs["dpt"], 2, 28, 28), 256),
        "ovg_camera_forward": (lambda ws, n: lib.ovg_camera_forward(hs["camera"], PTR, 1, 2, 4, PTR, ws, n, None),
                               lib.ovg_camera_workspace_bytes(hs["camera"], 2), 256),
    }


def outcomes():
    """{case: {"need": bytes, "null" / "misaligned" / "short": [return code, launches made, last error]}}; the cases in MISUSE
    get a well-formed workspace instead ("well-formed")."""
    from omnivggt_official_b200 import _lib as L
    lib = L.load()
    out = {}
    for name, (call, need, align) in cases(lib, L).items():
        res = {"need": need}
        bad = (("null", None, need), ("misaligned", PTR + align // 2, need), ("short", PTR, need - 1))
        for what, ws, n in (("well-formed", PTR, need),) if name in MISUSE else bad:
            before = lib.ovg_launch_count()
            rc = call(ws, n)
            res[what] = [rc, lib.ovg_launch_count() - before, lib.ovg_last_error().decode()]
        out[name] = res
    return out


@pytest.fixture(scope="module")
def refused():
    """outcomes() in a child process that sees no CUDA device."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    driver = ("import json, sys\n"
              f"sys.path[:0] = [{ROOT!r}, {TESTS!r}]\n"
              "import test_workspace_contract_cpu as t\n"
              "print(json.dumps(t.outcomes()))\n")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, "-c", driver], capture_output=True, text=True, timeout=600, cwd=TESTS, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


NAMES = ["ovg_point_cloud_count", "ovg_point_cloud_gather", "ovg_point_cloud_center", "ovg_point_cloud_scale", "ovg_match_index",
         "ovg_match_query", "ovg_match_gather", "ovg_match_pair", "ovg_tracks_assign", "ovg_tracks_assign(match)",
         "ovg_tracks_gather", "ovg_tracks_gather(match)", "ovg_bundle_adjust", "ovg_mesh_count", "ovg_mesh_faces",
         "ovg_mesh_compact", "ovg_tsdf_bounds", "ovg_tsdf_integrate", "ovg_tsdf_count", "ovg_tsdf_extract", "ovg_segment_sky",
         "ovg_farthest_point_sample", "ovg_compute_ranking", "ovg_sim3_estimate", "ovg_aggregator_forward",
         "ovg_aggregator_forward(layers)", "ovg_aggregator_forward(cp)", "ovg_dino_forward", "ovg_dpt_forward",
         "ovg_dpt_forward(f32)", "ovg_camera_forward"]
# argument combinations an entry point refuses before it looks at the workspace -> the reason it gives
MISUSE = {"ovg_aggregator_forward(cp, layers)": "no layer export",
          "ovg_aggregator_forward(depth_idx_local, no cp)": "need context parallelism",
          "ovg_dpt_forward(slots_f32 = 2)": "slots_f32 must be 0"}


def test_every_case_and_misuse_ran(refused):
    assert sorted(refused) == sorted(NAMES + list(MISUSE))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("what", ["null", "misaligned", "short"])
def test_bad_workspace_is_refused_before_any_launch(refused, name, what):
    r = refused[name]
    assert r["need"] > 0
    rc, launches, err = r[what]
    assert (rc, launches) == (OVG_E_INVALID, 0), err


@pytest.mark.parametrize("name", list(MISUSE))
def test_argument_misuse_is_refused(refused, name):
    rc, launches, err = refused[name]["well-formed"]
    assert (rc, launches) == (OVG_E_INVALID, 0) and MISUSE[name] in err, err
