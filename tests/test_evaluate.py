"""scene.evaluate (OmniVGGT.evaluate): the oracle's properties, the call sequence and argument errors on the host, the workspace
contract of the ovg_eval_* entry points, and on the H100 the device against the fp64 oracle (oracle/eval_oracle.py) on seeded
synthetic scenes: look-at cameras around a sphere, ground-truth depth ray-cast from them."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import eval_oracle as EO
from ovg_support import install

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)


# ------------------------------------------------------------------------------------------------------------------ scenes
def look_at(eye, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    """World-to-camera [3, 4] (x right, y down, z forward) of a camera at eye looking at target."""
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(z, -up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return np.concatenate([R, (-R @ eye)[:, None]], 1)


def sphere_scene(S, H, W, seed=0, radius=1.0):
    """(ext fp32 [S, 3, 4], intr fp32 [S, 3, 3], depth fp32 [S, H, W]): S cameras on a jittered ring around a unit sphere,
    the depth of each pixel ray-cast onto the sphere (0 where the ray misses)."""
    rng = np.random.default_rng(seed)
    ext, intr, depth = [], [], []
    f = 0.9 * W
    K = np.array([[f, 0, (W - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1]])
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    for s in range(S):
        a = 2 * math.pi * s / S + rng.normal(0, 0.05)
        eye = np.array([3.0 * math.cos(a), rng.normal(0, 0.5), 3.0 * math.sin(a)])
        E = look_at(eye, target=rng.normal(0, 0.05, 3))
        R, c = E[:, :3], eye
        d = np.stack([(u - K[0, 2]) / f, (v - K[1, 2]) / f, np.ones_like(u)], -1) @ R      # world ray per unit depth
        a2 = (d * d).sum(-1)
        b = 2 * (d @ c)
        disc = b * b - 4 * a2 * (c @ c - radius ** 2)
        z = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a2), 0.0)
        ext.append(E)
        intr.append(K)
        depth.append(z)
    return np.array(ext, np.float32), np.array(intr, np.float32), np.array(depth, np.float32)


def sim3_of(rng):
    """A random similarity (s, R, t)."""
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    return float(rng.uniform(0.5, 2.0)), R, rng.normal(size=3)


def transform_cameras(ext, s, R, t):
    """World-to-camera extrinsics of the same cameras in the world x' = s R x + t."""
    out = []
    for E in np.asarray(ext, np.float64):
        Rc, tc = E[:, :3], E[:, 3]
        Rn = Rc @ R.T
        out.append(np.concatenate([Rn, (s * tc - Rn @ t)[:, None]], 1))
    return np.array(out)


def rot_y(deg):
    a = math.radians(deg)
    return np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])


# ------------------------------------------------------------------------------------------------------------------ oracle
def test_oracle_perfect_prediction_scores_perfectly():
    ext, intr, depth = sphere_scene(6, 40, 48, seed=1)
    pose = EO.pose_metrics(ext, intr, ext)
    assert pose["n"] == 6 and abs(pose["ate"]) < 1e-6
    assert np.abs(pose["rpe"]).max() < 1e-5
    assert (pose["auc"] == 1).all() and (pose["rra"] == 1).all() and (pose["rta"] == 1).all()
    d = EO.depth_metrics(depth, depth)
    assert d["abs_rel"] == 0 and (d["delta"] == 1).all() and d["scale"] == 1
    pts = EO.unproject(depth, ext, intr).astype(np.float32)
    keep = depth > 0
    p = EO.point_metrics(pts, pts, keep)
    assert p["acc"] == 0 and p["comp"] == 0 and abs(p["nc"] - 1) < 1e-12


def test_oracle_planted_sim3_is_aligned_away():
    rng = np.random.default_rng(2)
    ext, intr, depth = sphere_scene(6, 40, 48, seed=2)
    s, R, t = sim3_of(rng)
    pred_ext = transform_cameras(ext, s, R, t)
    pose = EO.pose_metrics(ext, intr, pred_ext)
    gt_pose = EO.pose_metrics(ext, intr, ext)
    assert abs(pose["ate"]) < 1e-6 and np.abs(pose["rpe"]).max() < 1e-5        # fp32 centres feed the fit
    np.testing.assert_allclose(pose["pair_errors"], gt_pose["pair_errors"], atol=1e-4)
    assert (pose["auc"] == 1).all()
    d = EO.depth_metrics(depth, (depth * s).astype(np.float32))
    assert abs(d["abs_rel"]) < 1e-7 and (d["delta"] == 1).all()
    pts = EO.unproject(depth, ext, intr)
    A, t_fit, c, rms = EO.umeyama((pts[depth > 0] * s) @ R.T + t, pts[depth > 0])
    assert rms < 1e-9 and abs(c * s - 1) < 1e-9


def test_oracle_planted_rotation_gives_its_rre():
    ext = np.array([look_at((3.0 * math.cos(a), 0.3 * a, 3.0 * math.sin(a))) for a in (0.0, 1.0, 2.5)])    # fp64: orthonormal
    pred = ext.copy()
    Ry = rot_y(10.0)
    pred[1, :, :3] = Ry @ pred[1, :, :3]               # about the camera's own y axis: the centre stays
    pred[1, :, 3] = Ry @ pred[1, :, 3]
    _, rre, rte = EO.pair_errors(ext, pred)
    assert abs(rre[0] - 10.0) < 1e-9 and abs(rre[2] - 10.0) < 1e-9 and abs(rre[1]) < 1e-4


def test_oracle_nearest_neighbours_are_brute_force():
    rng = np.random.default_rng(4)
    a, b = rng.normal(size=(300, 3)), rng.normal(size=(200, 3))
    d, i = EO.nearest(a, b)
    full = np.sqrt(((a[:, None] - b[None]) ** 2).sum(-1))
    assert (i == full.argmin(1)).all()
    np.testing.assert_allclose(d, full.min(1), rtol=1e-15)


def test_oracle_rpe_on_a_hand_built_trajectory():
    # three camera-to-world poses: identity, a unit step along x, then a 90 degree turn about z in place
    Rz = np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 1]])
    Rq = np.array([np.eye(3), np.eye(3), Rz])
    cq = np.array([[0.0, 0, 0], [1, 0, 0], [1, 0, 0]])
    # the prediction overshoots the step by 0.5 and turns by 80 degrees
    a = math.radians(80)
    Rp = np.array([np.eye(3), np.eye(3), [[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]]])
    cp = np.array([[0.0, 0, 0], [1.5, 0, 0], [1.5, 0, 0]])
    e = EO.rpe_errors(Rq, cq, Rp, cp)
    assert e.shape == (2, 2)                              # consecutive pairs (0, 1), (1, 2) only
    np.testing.assert_allclose(e[0], [0.5, 0.0], atol=1e-12)
    np.testing.assert_allclose(e[1], [0.0, 10.0], atol=1e-12)


def test_oracle_drops_loader_placeholder_views():
    ext, intr, _ = sphere_scene(5, 8, 8, seed=5)
    intr[2] = 0
    ext[2] = 0
    pose = EO.pose_metrics(ext, intr, ext)
    assert pose["n"] == 4 and list(pose["views"]) == [0, 1, 3, 4]
    assert not any(2 in p for p in pose["pairs"].tolist())


# ------------------------------------------------------------------------------------------------------------------ dry runs
def _dry_predictions(S=4, H=6, W=7):
    g = torch.Generator().manual_seed(0)
    return {"images": torch.rand(1, S, 3, H, W, generator=g), "depth": torch.rand(1, S, H, W, 1, generator=g) + 1,
            "world_points_from_depth": torch.randn(1, S, H, W, 3, generator=g),
            "extrinsic": torch.eye(4)[:3].repeat(1, S, 1, 1)}


def _dry_gt(S=4, H=6, W=7):
    ext, intr, depth = sphere_scene(S, H, W, seed=6)
    return dict(extrinsics=torch.from_numpy(ext)[None], intrinsics=torch.from_numpy(intr)[None],
                depth=torch.from_numpy(depth)[None, ..., None], mask=torch.ones(1, S, H, W))


def _read(t):
    """Host reads of a dry run: the fits' (count, status) as a good fit of 5, the matcher's counts as finite."""
    if t.dtype == torch.float64:
        return torch.tensor([5.0, 0.0])
    return torch.zeros_like(t, device="cpu")


@pytest.fixture()
def dry_eval(monkeypatch):
    return install(monkeypatch, read=_read)


ORDER = ["ovg_eval_pose_workspace_bytes", "ovg_eval_pose", "host_read", "ovg_eval_depth_workspace_bytes", "ovg_eval_depth",
         "ovg_eval_points_keep", "ovg_unproject_depth", "ovg_sim3_workspace_bytes", "ovg_sim3_estimate", "host_read",
         "ovg_sim3_apply", "ovg_match_workspace_bytes", "ovg_match_index", "ovg_match_query", "host_read",
         "ovg_eval_points_workspace_bytes", "ovg_eval_points"]


def test_dry_run_call_order_and_host_reads(dry_eval):
    from omnivggt_official_b200 import OmniVGGT
    out = OmniVGGT.evaluate(_dry_predictions(), **_dry_gt(), views=[3, 1, 2])
    assert dry_eval.names() == ORDER
    assert dry_eval.count("host_read") == 3
    assert set(out) == {"pose", "depth", "points"}
    # the match workspace goes from the matcher to ovg_eval_points
    (idx,) = dry_eval.args("ovg_match_index")
    (pts,) = dry_eval.args("ovg_eval_points")
    assert pts[5:7] == idx[5:7]
    # views: ascending, as int32 on the device for the pose group, a per-view selection for the others
    (pose,) = dry_eval.args("ovg_eval_pose")
    assert pose[4] == 3


def test_dry_run_groups_follow_the_ground_truth(dry_eval):
    from omnivggt_official_b200 import OmniVGGT
    gt = _dry_gt()
    out = OmniVGGT.evaluate(_dry_predictions(), depth=gt["depth"])
    assert set(out) == {"depth"} and dry_eval.names() == ["ovg_eval_depth_workspace_bytes", "ovg_eval_depth"]
    dry_eval.calls.clear()
    out = OmniVGGT.evaluate(_dry_predictions(), extrinsics=gt["extrinsics"], intrinsics=gt["intrinsics"])
    assert set(out) == {"pose"} and dry_eval.names() == ORDER[:3]


BAD = {
    "no ground truth": dict(),
    "extrinsics only": dict(extrinsics="ext"),
    "bad extrinsics shape": dict(extrinsics=torch.zeros(1, 4, 2, 4), intrinsics="intr"),
    "integer depth": dict(depth=torch.zeros(1, 4, 6, 7, dtype=torch.int32)),
    "depth at another size": dict(depth=torch.zeros(1, 4, 5, 7)),
    "views out of range": dict(depth="depth", views=[0, 4]),
    "views repeated": dict(depth="depth", views=[1, 1]),
    "views empty": dict(depth="depth", views=[]),
    "pointmap without world_points": dict(extrinsics="ext", intrinsics="intr", depth="depth", source="pointmap"),
    "bad source": dict(depth="depth", source="cloud"),
    "mask without depth": dict(mask="mask"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_argument_errors_before_any_library_call(dry_eval, case):
    from omnivggt_official_b200 import OmniVGGT
    gt = _dry_gt()
    names = {"ext": gt["extrinsics"], "intr": gt["intrinsics"], "depth": gt["depth"], "mask": gt["mask"]}
    kw = {k: names.get(v, v) if isinstance(v, str) and k != "source" else v for k, v in BAD[case].items()}
    with pytest.raises(ValueError):
        OmniVGGT.evaluate(_dry_predictions(), **kw)
    assert dry_eval.calls == []


def test_too_many_camera_views_and_pixels_are_refused(dry_eval):
    from omnivggt_official_b200 import scene
    S = scene.EVAL_MAX_CAMERA_VIEWS + 1
    pred = {"images": torch.zeros(1, S, 3, 1, 1), "extrinsic": torch.zeros(1, S, 3, 4)}
    with pytest.raises(ValueError, match="at most 8192"):
        scene.evaluate(pred, extrinsics=torch.zeros(S, 3, 4), intrinsics=torch.zeros(S, 3, 3))
    big = {"images": torch.zeros(1, 2, 3, 1, 1).expand(1, 2, 3, 2 ** 15, 2 ** 15)}
    with pytest.raises(ValueError, match="2\\^31"):
        scene.evaluate(big, depth=torch.zeros(1, 2, 1, 1).expand(1, 2, 2 ** 15, 2 ** 15))
    assert dry_eval.calls == []


# ------------------------------------------------------------------------------------------------------------------ workspaces
OVG_E_INVALID = -1
PTR = 1 << 40
S_, H_, W_ = 3, 8, 8


def contract_cases(lib):
    """{entry: (call(workspace, bytes), bytes needed)}; "(match)" breaks the match workspace of ovg_eval_points."""
    match_need = lib.ovg_match_workspace_bytes(2, S_ * H_ * W_, 1)
    pts_need = lib.ovg_eval_points_workspace_bytes(S_, H_, W_)

    def points(mws, mwsb, ws, wsb):
        return lib.ovg_eval_points(PTR, PTR, S_, H_, W_, mws, mwsb, ws, wsb, PTR, PTR, PTR, None)

    return {
        "ovg_eval_pose": (lambda ws, n: lib.ovg_eval_pose(PTR, PTR, PTR, PTR, S_, ws, n, *([PTR] * 6), None),
                          lib.ovg_eval_pose_workspace_bytes(S_)),
        "ovg_eval_depth": (lambda ws, n: lib.ovg_eval_depth(PTR, None, PTR, PTR, S_, H_ * W_, ws, n, PTR, PTR, PTR, PTR, None),
                           lib.ovg_eval_depth_workspace_bytes(S_, H_ * W_)),
        "ovg_eval_points": (lambda ws, n: points(PTR, match_need, ws, n), pts_need),
        "ovg_eval_points(match)": (lambda ws, n: points(ws, n, PTR, pts_need), match_need),
    }


def contract_outcomes():
    from omnivggt_official_b200 import _lib as L
    lib = L.load()
    out = {}
    for name, (call, need) in contract_cases(lib).items():
        res = {"need": need}
        for what, ws, n in (("null", None, need), ("misaligned", PTR + 128, need), ("short", PTR, need - 1)):
            before = lib.ovg_launch_count()
            rc = call(ws, n)
            res[what] = [rc, lib.ovg_launch_count() - before, lib.ovg_last_error().decode()]
        out[name] = res
    return out


@pytest.fixture(scope="module")
def refused():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    driver = ("import json, sys\n"
              f"sys.path[:0] = [{ROOT!r}, {TESTS!r}]\n"
              "import test_evaluate as t\n"
              "print(json.dumps(t.contract_outcomes()))\n")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, "-c", driver], capture_output=True, text=True, timeout=600, cwd=TESTS, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", ["ovg_eval_pose", "ovg_eval_depth", "ovg_eval_points", "ovg_eval_points(match)"])
@pytest.mark.parametrize("what", ["null", "misaligned", "short"])
def test_bad_workspace_is_refused_before_any_launch(refused, name, what):
    r = refused[name]
    assert r["need"] > 0
    rc, launches, err = r[what]
    assert (rc, launches) == (OVG_E_INVALID, 0), err


# ------------------------------------------------------------------------------------------------------------------ GPU
def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pose_case(n, seed):
    """(gt ext, intr, predicted ext): a ring of n cameras and a noisy, similarity-transformed prediction."""
    rng = np.random.default_rng(seed)
    ext, intr, _ = sphere_scene(n, 4, 4, seed=seed)
    s, R, t = sim3_of(rng)
    pred = transform_cameras(ext, s, R, t)
    for k in range(n):                                    # rotation noise, and centre noise through t
        a = rng.normal(0, 0.03, 3)
        th = np.linalg.norm(a)
        Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]) / th
        dR = np.eye(3) + math.sin(th) * Kx + (1 - math.cos(th)) * Kx @ Kx
        pred[k, :, :3] = dR @ pred[k, :, :3]
        pred[k, :, 3] = pred[k, :, 3] + rng.normal(0, 0.05, 3)
    return ext, intr, pred.astype(np.float32)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _pred(S, H, W, **kw):
    return dict({"images": torch.zeros(1, S, 3, H, W, device="cuda")}, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 24, 300, 1000])
def test_pose_against_the_oracle(n):
    from omnivggt_official_b200 import OmniVGGT
    ext, intr, pred = _pose_case(n, seed=n)
    out = OmniVGGT.evaluate(_pred(n, 4, 4, extrinsic=_cuda(pred)[None]), extrinsics=_cuda(ext)[None],
                            intrinsics=_cuda(intr)[None])["pose"]
    ref = EO.pose_metrics(ext, intr, pred)
    assert int(out["views"]) == n
    assert _rel(out["sim3"].cpu(), ref["sim3"]) < 1e-9
    for k in ("ate", "rpe_trans", "rpe_rot"):
        assert _rel(float(out[k]), ref[k]) < 1e-9, k
    given = EO.pose_metrics(ext, intr, pred, sim3=out["sim3"].cpu().numpy())
    assert np.abs(out["rpe_errors"].cpu().numpy() - given["rpe"]).max() < 1e-9
    perr = out["pair_errors"].cpu().numpy()
    assert (out["pairs"].cpu().numpy() == ref["pairs"]).all()
    assert np.abs(perr - ref["pair_errors"]).max() < 1e-9
    own = EO.pair_scores(perr[:, 0], perr[:, 1])            # the protocol on the device's own errors: exact
    for k in ("auc", "rra", "rta"):
        assert (out[k].cpu().numpy() == own[k]).all(), k
        assert np.abs(out[k].cpu().numpy() - ref[k]).max() <= 1.0 / len(perr) + 1e-15, k


def _depth_case(S, H, W, seed):
    rng = np.random.default_rng(seed)
    ext, intr, depth = sphere_scene(S, H, W, seed=seed)
    pred = (depth * 0.37 * np.exp(rng.normal(0, 0.1, depth.shape))).astype(np.float32)
    pred[depth == 0] = rng.uniform(0, 5, (depth == 0).sum())
    mask = rng.uniform(size=depth.shape) > 0.05
    return ext, intr, depth, pred, mask


@pytest.mark.gpu
def test_depth_against_the_oracle():
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = 24, 518, 518
    ext, intr, depth, pred, mask = _depth_case(S, H, W, seed=7)
    views = list(range(1, S, 2))
    out = OmniVGGT.evaluate(_pred(S, H, W, depth=_cuda(pred)[None, ..., None]), depth=_cuda(depth)[None],
                            mask=_cuda(mask)[None], views=views)["depth"]
    ref = EO.depth_metrics(depth, pred, mask, views)
    assert int(out["pixels"]) == ref["pixels"] > 0
    for k in ("median_gt", "median_pred", "scale"):
        assert float(out[k]) == float(ref[k]), k
    assert (np.rint(out["delta"].cpu().numpy() * ref["pixels"]) == ref["delta_counts"]).all()
    for k in ("abs_rel", "sq_rel", "rmse"):
        assert _rel(float(out[k]), ref[k]) < 1e-12, k
    assert _rel(out["delta"].cpu(), ref["delta"]) < 1e-15
    assert (out["view_pixels"].cpu().numpy() == ref["view_pixels"]).all()
    for k in ("view_abs_rel", "view_delta1"):
        got = out[k].cpu().numpy()
        assert (np.isnan(got) == np.isnan(ref[k])).all() and np.isnan(got[0]), k
        ok = ~np.isnan(got)
        assert _rel(got[ok], ref[k][ok]) < 1e-12, k


@pytest.mark.gpu
def test_depth_without_valid_pixels_is_nan():
    from omnivggt_official_b200 import OmniVGGT
    out = OmniVGGT.evaluate(_pred(2, 8, 8, depth=torch.ones(1, 2, 8, 8, device="cuda")),
                            depth=torch.zeros(1, 2, 8, 8, device="cuda"))["depth"]
    assert int(out["pixels"]) == 0 and math.isnan(float(out["abs_rel"])) and math.isnan(float(out["scale"]))


def _points_case(S, H, W, seed):
    """Ground truth of a sphere scene, and a prediction whose cameras and points are a noisy similarity of it."""
    rng = np.random.default_rng(seed)
    ext, intr, depth = sphere_scene(S, H, W, seed=seed)
    s, R, t = sim3_of(rng)
    pts = EO.unproject(depth, ext, intr)
    pts = (s * pts @ R.T + t + rng.normal(0, 0.002, pts.shape)).astype(np.float32)
    pts[depth == 0] = np.nan
    pred_ext = transform_cameras(ext, s, R, t).astype(np.float32)
    return ext, intr, depth, pts, pred_ext


def _device_clouds(ext, intr, depth, pts, sim3, views=None):
    """The ground-truth points and the shared set the device uses, and the prediction aligned by the documented rounding."""
    from omnivggt_official_b200 import ops
    S, H, W = depth.shape
    sel = torch.zeros(S, dtype=torch.uint8)
    sel[list(range(S)) if views is None else views] = 1
    gd = _cuda(depth).view(S, H * W)
    c2w, keep = ops.eval_points_keep(_cuda(ext), _cuda(intr), gd, None, _cuda(pts).view(S, H * W, 3), sel.cuda())
    gt = ops.unproject_depth(gd.view(S, H, W), _cuda(intr), c2w, H, W).cpu().numpy()
    return gt, keep[0].view(S, H, W).bool().cpu().numpy(), EO.sim3_apply(sim3, pts)


def _check_points(out, ext, intr, depth, pts, views=None):
    gt, keep, aligned = _device_clouds(ext, intr, depth, pts, out["sim3"].cpu().numpy(), views)
    ok = EO.depth_valid(depth, depth, None, views) & np.isfinite(pts).all(-1) & EO.camera_ok(ext, intr)[:, None, None]
    assert (keep == ok).all()
    A, t, _, _ = EO.umeyama(pts[keep], gt[keep])
    fit = np.eye(4)
    fit[:3, :3], fit[:3, 3] = A, t
    assert _rel(out["sim3"].cpu().numpy(), fit) < 1e-9
    ref = EO.point_metrics(aligned, gt, keep)
    assert int(out["pixels"]) == ref["pixels"]
    assert (out["acc_dist"].cpu().numpy() == ref["acc_dist"]).all()
    assert (out["comp_dist"].cpu().numpy() == ref["comp_dist"]).all()
    for k in ("acc_median", "comp_median"):
        assert float(out[k]) == float(ref[k]), k
    for k in ("acc", "comp", "chamfer", "nc_acc", "nc_comp", "nc"):
        if np.isnan(ref[k]):                                   # no point with a normal: NaN on both sides
            assert math.isnan(float(out[k])), k
        else:
            assert _rel(float(out[k]), ref[k]) < 1e-12, k


@pytest.mark.gpu
@pytest.mark.parametrize("S", [8, 24])
def test_points_against_the_oracle(S):
    from omnivggt_official_b200 import OmniVGGT
    H = W = 518
    ext, intr, depth, pts, pred_ext = _points_case(S, H, W, seed=S)
    pred = _pred(S, H, W, extrinsic=_cuda(pred_ext)[None], depth=_cuda(depth)[None], world_points_from_depth=_cuda(pts)[None])
    out = OmniVGGT.evaluate(pred, extrinsics=_cuda(ext)[None], intrinsics=_cuda(intr)[None], depth=_cuda(depth)[None])
    _check_points(out["points"], ext, intr, depth, pts)
    assert 0.9 < float(out["points"]["nc"]) <= 1.0
    assert float(out["pose"]["ate"]) < 1e-4 and float(out["pose"]["auc"][0]) == 1.0


@pytest.mark.gpu
def test_placeholders_and_views_restrict_every_group():
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = 6, 64, 80
    ext, intr, depth, pts, pred_ext = _points_case(S, H, W, seed=11)
    ext[2], intr[2] = 0, 0                                   # the loader's placeholder for a view without a camera
    pred = _pred(S, H, W, extrinsic=_cuda(pred_ext)[None], depth=_cuda(depth)[None], world_points_from_depth=_cuda(pts)[None])
    views = [0, 2, 3, 5]
    out = OmniVGGT.evaluate(pred, extrinsics=_cuda(ext)[None], intrinsics=_cuda(intr)[None], depth=_cuda(depth)[None],
                            views=views)
    ref = EO.pose_metrics(ext, intr, pred_ext, views)
    assert int(out["pose"]["views"]) == 3 and (out["pose"]["pairs"].cpu().numpy() == ref["pairs"]).all()
    assert (out["depth"]["view_pixels"].cpu().numpy()[[1, 4]] == 0).all()
    assert out["depth"]["view_pixels"].cpu().numpy()[2] > 0       # depth needs no camera
    _check_points(out["points"], ext, intr, depth, pts, views)


def _flat(d, path=""):
    if isinstance(d, dict):
        return [x for k in sorted(d) for x in _flat(d[k], f"{path}.{k}")]
    return [(path, d)]


@pytest.mark.gpu
def test_bit_identical_across_calls_and_under_poison():
    from omnivggt_official_b200 import OmniVGGT
    from test_poison_gpu import check_case
    S, H, W = 8, 96, 128
    ext, intr, depth, pts, pred_ext = _points_case(S, H, W, seed=13)
    args = [_cuda(a)[None] for a in (ext, intr, depth, pts, pred_ext)]

    def run(P):
        pred = _pred(S, H, W, extrinsic=args[4], depth=args[2], world_points_from_depth=args[3])
        return OmniVGGT.evaluate(pred, extrinsics=args[0], intrinsics=args[1], depth=args[2])

    a, b = _flat(run(None)), _flat(run(None))
    for (pa, x), (_, y) in zip(a, b):
        assert x.dtype == y.dtype and torch.equal(x.reshape(-1).view(torch.uint8), y.reshape(-1).view(torch.uint8)), pa
    check_case("evaluate", run)


@pytest.mark.gpu
def test_mini_model_forward_and_reconstruct():
    from omnivggt_official_b200 import OmniVGGT
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    H = W = 56
    inp = {k: v.cuda() for k, v in make_inputs(1, 4, H, W, seed=4).items()}
    pred = m.postprocess(m(depth_gt_index=[1], camera_gt_index=[0], **inp))
    rec = m.reconstruct(**{k: v.cuda() for k, v in make_inputs(1, 10, H, W, seed=63).items()}, chunk=6, overlap=2)
    for p in (pred, rec):
        S = p["depth"].shape[1]
        ext, intr, depth = sphere_scene(S, H, W, seed=17)
        gt = dict(extrinsics=_cuda(ext)[None], intrinsics=_cuda(intr)[None], depth=_cuda(depth)[None])
        pe = p["extrinsic"][0].float().cpu().numpy()
        views = list(range(1, S))
        try:
            ref = EO.pose_metrics(ext, intr, pe, views)
        except ValueError:
            with pytest.raises(ValueError):
                OmniVGGT.evaluate(p, views=views, **gt)
            continue
        out = OmniVGGT.evaluate(p, views=views, **gt)
        assert _rel(float(out["pose"]["ate"]), ref["ate"]) < 1e-9
        assert np.abs(out["pose"]["pair_errors"].cpu().numpy() - ref["pair_errors"]).max() < 1e-9
        dref = EO.depth_metrics(depth, p["depth"][0, ..., 0].float().cpu().numpy(), None, views)
        assert float(out["depth"]["scale"]) == float(dref["scale"])
        assert _rel(float(out["depth"]["abs_rel"]), dref["abs_rel"]) < 1e-12
        pts = p["world_points_from_depth"][0].float().cpu().numpy()
        _check_points(out["points"], ext, intr, depth, pts, views)
