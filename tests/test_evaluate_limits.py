"""scene.evaluate at its limits: dry runs at pixel counts that are not a multiple of 4 and with ground truth at an odd storage
offset, the per-group size refusals, and on the H100 the device against the fp64 oracle (oracle/eval_oracle.py) past one
1024-view compaction round up to the 8192-view limit, at more than 65535 depth views, past 2 GiB of depth selection columns,
at odd shapes and exactly on the thresholds."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import eval_oracle as EO
from ovg_support import install
from test_evaluate import (ORDER, _check_points, _cuda, _dry_gt, _dry_predictions, _points_case, _pose_case, _pred, _read,
                           _rel, rot_y, sphere_scene)


# ------------------------------------------------------------------------------------------------------------------ dry runs
def _floats(ptr, n):
    return np.ctypeslib.as_array((C.c_float * n).from_address(ptr))


def _aligned_dry(monkeypatch, S, H, W):
    """A dry run whose ovg_unproject_depth checks the alignment ovg.h documents, copies the depth it is given and writes a
    known pattern; ovg_sim3_estimate records the ground-truth cloud it is handed (dst)."""
    seen = {}

    def unproject(a):
        depth, _, _, world, K, h, w = a[:7]
        assert depth % 16 == 0 and world % 16 == 0, "ovg_unproject_depth needs 16-byte aligned depth and world"
        seen["depth"] = _floats(depth, K * h * w).copy()
        _floats(world, K * h * w * 3)[:] = np.arange(K * h * w * 3, dtype=np.float32)

    def estimate(a):
        seen["dst"] = _floats(a[1], S * H * W * 3).copy()

    fake = install(monkeypatch, read=_read, effects={"ovg_unproject_depth": unproject, "ovg_sim3_estimate": estimate})
    return fake, seen


@pytest.mark.parametrize("shape", [(3, 5, 7), (6, 5, 7), (5, 5, 7)], ids=["1mod4", "2mod4", "3mod4"])
@pytest.mark.parametrize("offset", [False, True], ids=["dense", "odd_offset_depth"])
def test_dry_run_unprojects_aligned_at_any_pixel_count(monkeypatch, shape, offset):
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = shape
    fake, seen = _aligned_dry(monkeypatch, S, H, W)
    gt = _dry_gt(S, H, W)
    depth = gt["depth"]
    if offset:                                   # a view one float into its storage: 4 bytes past 16-byte alignment
        buf = torch.zeros(depth.numel() + 1)
        buf[1:] = depth.reshape(-1)
        gt["depth"] = buf[1:].view(depth.shape)
        assert gt["depth"].data_ptr() % 16 == 4
    OmniVGGT.evaluate(_dry_predictions(S, H, W), **gt, views=list(range(S)))
    assert fake.names() == ORDER
    np.testing.assert_array_equal(seen["depth"], depth.reshape(-1).numpy())
    # the ground-truth cloud that reaches the fit is exactly what the unprojection wrote
    np.testing.assert_array_equal(seen["dst"], np.arange(S * H * W * 3, dtype=np.float32))


def _zeros(*shape):
    return torch.zeros((1,) * len(shape)).expand(*shape)


POINT_LIMITS = {"2^30 pixels": (2, 2 ** 14, 2 ** 15), "just below 2^31": (2 ** 15 - 1, 2 ** 8, 2 ** 8),
                "65536 views": (65536, 1, 1)}


@pytest.mark.parametrize("case", sorted(POINT_LIMITS))
def test_points_group_limits_are_refused_before_any_library_call(dry_eval, case):
    from omnivggt_official_b200 import scene
    S, H, W = POINT_LIMITS[case]
    assert S * H * W < 2 ** 31 and (S * H * W >= 2 ** 30 or S > 65535)
    pred = {"images": _zeros(1, S, 3, H, W), "extrinsic": _zeros(1, S, 3, 4), "depth": _zeros(1, S, H, W),
            "world_points_from_depth": _zeros(1, S, H, W, 3)}
    with pytest.raises(ValueError, match="points group"):
        scene.evaluate(pred, extrinsics=_zeros(S, 3, 4), intrinsics=_zeros(S, 3, 3), depth=_zeros(1, S, H, W), views=[0, 1])
    assert dry_eval.calls == []


@pytest.mark.parametrize("case", sorted(POINT_LIMITS))
def test_depth_only_scene_of_the_same_size_reaches_the_library(dry_eval, case):
    """The limits are the points group's: the depth group alone runs at these sizes (on meta tensors: nothing is allocated)."""
    from omnivggt_official_b200 import scene
    S, H, W = POINT_LIMITS[case]

    def meta(*shape):
        return torch.zeros((1,) * len(shape), device="meta").expand(*shape)

    out = scene.evaluate({"images": meta(1, S, 3, H, W), "depth": meta(1, S, H, W)}, depth=meta(1, S, H, W))
    assert set(out) == {"depth"}
    assert dry_eval.names() == ["ovg_eval_depth_workspace_bytes", "ovg_eval_depth"]
    (args,) = dry_eval.args("ovg_eval_depth")
    assert args[4:6] == (S, H * W)


@pytest.fixture()
def dry_eval(monkeypatch):
    return install(monkeypatch, read=_read)


def test_oracle_drops_views_whose_centre_overflows_fp32():
    ext, intr, _ = sphere_scene(6, 4, 4, seed=3)
    pred = ext.copy()
    ext[1] = _overflowing(ext[1])
    pred[4] = _overflowing(pred[4])
    assert np.isfinite(ext).all() and np.isfinite(pred).all()
    out = EO.pose_metrics(ext, intr, pred)
    assert out["n"] == 4 and list(out["views"]) == [0, 2, 3, 5] and np.isfinite(out["ate"])


def test_chunked_oracles_match_the_whole():
    ext, intr, pred = _pose_case(40, seed=5)
    a, b = EO.pose_metrics(ext, intr, pred), EO.pose_metrics(ext, intr, pred, chunk=97)
    assert (a["pairs"] == b["pairs"]).all() and (a["pair_errors"] == b["pair_errors"]).all()
    for k in ("auc", "rra", "rta"):
        assert (a[k] == b[k]).all()
    rng = np.random.default_rng(1)
    g = rng.uniform(0.5, 4, (7, 9, 11)).astype(np.float32)
    p = (g * rng.uniform(0.7, 1.4, g.shape)).astype(np.float32)
    mask = rng.uniform(size=g.shape) > 0.2
    a, b = EO.depth_metrics(g, p, mask, [0, 2, 3, 6]), EO.depth_metrics(g, p, mask, [0, 2, 3, 6], chunk=3)
    _check_depth_dicts(b, a)


# ------------------------------------------------------------------------------------------------------------------ helpers
def _overflowing(E):
    """A finite world-to-camera [3, 4] whose centre -R^T t overflows fp32: R about z by 45 degrees, t = (3e38, 3e38, 0)."""
    c, s = np.cos(np.pi / 4), np.sin(np.pi / 4)
    out = np.array(E, np.float32)
    out[:, :3] = [[c, -s, 0], [s, c, 0], [0, 0, 1]]
    out[:, 3] = [3e38, 3e38, 0]
    return out


def _same(a, b):
    """Equal values, NaN where the other is NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(((a == b) | (np.isnan(a) & np.isnan(b))).all())


def _close(a, b, rtol=1e-12):
    """The same NaN and infinities, finite values within rtol of the largest."""
    a, b = np.atleast_1d(np.asarray(a, np.float64)), np.atleast_1d(np.asarray(b, np.float64))
    if a.shape != b.shape or not (np.isnan(a) == np.isnan(b)).all():
        return False
    fin = np.isfinite(b)
    if not (a[~fin & ~np.isnan(b)] == b[~fin & ~np.isnan(b)]).all() or not np.isfinite(a[fin]).all():
        return False
    return not fin.any() or _rel(a[fin], b[fin]) <= rtol


def _check_depth_dicts(out, ref):
    """A depth group (device tensors or an oracle dict) against the oracle."""
    host = {k: (v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()}
    assert int(host["pixels"]) == ref["pixels"]
    for k in ("median_gt", "median_pred", "scale"):
        assert _same(host[k], ref[k]), (k, host[k], ref[k])
    if ref["pixels"]:
        counts = host["delta_counts"] if "delta_counts" in host else np.rint(host["delta"] * ref["pixels"])
        assert (counts == ref["delta_counts"]).all(), (counts, ref["delta_counts"])
    assert _same(host["delta"], ref["delta"])
    for k in ("abs_rel", "sq_rel", "rmse", "view_abs_rel", "view_delta1"):
        assert _close(host[k], ref[k]), (k, host[k], ref[k])
    assert (host["view_pixels"] == ref["view_pixels"]).all()


# ------------------------------------------------------------------------------------------------------------------ GPU: pose
DROP_AT = (0, 1023, 1024, 2047, 2048, -1)


def _drop(ext, intr, pred, v, how):
    if how == "placeholder":                        # the loader's view without a camera
        ext[v], intr[v] = 0, 0
    elif how == "pred_nan":
        pred[v, 1, 2] = np.nan
    else:
        ext[v, 0, 3] = np.inf


def _flat_bits(out):
    return {k: v.reshape(-1).view(torch.uint8).clone() for k, v in out.items()}


def _check_pose(out, ext, intr, pred, views=None, chunk=None, atol=0.0):
    """The device's pose group against the oracle; returns the oracle's result.  ``atol`` is added to the 1e-9 relative
    tolerance of the ATE and RPE, for the edge cases where some of them are 0 up to rounding."""
    ref = EO.pose_metrics(ext, intr, pred, views, chunk=chunk)
    n = ref["n"]
    assert int(out["views"]) == n
    pairs = out["pairs"].cpu().numpy()
    assert pairs.shape == (n * (n - 1) // 2, 2) and (pairs == ref["pairs"]).all()
    assert _rel(out["sim3"].cpu(), ref["sim3"]) < 1e-9
    for k in ("ate", "rpe_trans", "rpe_rot"):
        assert abs(float(out[k]) - ref[k]) <= 1e-9 * abs(ref[k]) + atol, k
    rpe = out["rpe_errors"].cpu().numpy()
    assert rpe.shape == (n - 1, 2) and np.abs(rpe - ref["rpe"]).max() < 1e-9
    perr = out["pair_errors"].cpu().numpy()
    assert np.abs(perr - ref["pair_errors"]).max() < 1e-9
    own = EO.pair_scores(perr[:, 0], perr[:, 1])
    for k in ("auc", "rra", "rta"):
        got = out[k].cpu().numpy()
        assert (got == own[k]).all(), k
        assert np.abs(got - ref[k]).max() <= 1.0 / len(perr) + 1e-15, k
    return ref


POSE_LIMIT_CASES = [1023, 1024, 1025, 2047, 2049, 4096, 8192, "8192 of 9000"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", POSE_LIMIT_CASES, ids=str)
def test_pose_past_one_compaction_round_against_the_oracle(case):
    from omnivggt_official_b200 import OmniVGGT
    S = 9000 if isinstance(case, str) else case
    ext, intr, pred = _pose_case(S, seed=S)
    views = None
    if isinstance(case, str):
        views = sorted(np.random.default_rng(9).choice(S, 8192, replace=False).tolist())
    scored = list(range(S)) if views is None else views
    positions = sorted({p % len(scored) for p in DROP_AT if p < len(scored)})
    for k, pos in enumerate(positions):          # each position dropped one of three ways, the way shifting with the case
        _drop(ext, intr, pred, scored[pos], ("placeholder", "pred_nan", "gt_inf")[(k + POSE_LIMIT_CASES.index(case)) % 3])
    pe = _pred(S, 4, 4, extrinsic=_cuda(pred)[None])
    gt = dict(extrinsics=_cuda(ext)[None], intrinsics=_cuda(intr)[None])
    out = OmniVGGT.evaluate(pe, **gt, views=views)["pose"]
    ref = _check_pose(out, ext, intr, pred, views, chunk=1 << 21)
    assert ref["n"] == len(scored) - len(positions)
    assert not set(scored[p] for p in positions) & set(ref["views"].tolist())
    again = OmniVGGT.evaluate(pe, **gt, views=views)["pose"]
    a, b = _flat_bits(out), _flat_bits(again)
    assert all(torch.equal(a[k], b[k]) for k in a)


def _ring(n, seed):
    """World-to-camera fp32 [n, 3, 4] of look-at cameras on a ring, intrinsics, and a noisy similarity of them."""
    ext, intr, pred = _pose_case(n, seed)
    return ext.copy(), intr, pred.copy()


def _identity_cams(n, seed):
    """Cameras with the identity rotation (so relative rotations are exactly I) at random centres."""
    rng = np.random.default_rng(seed)
    ext = np.zeros((n, 3, 4), np.float32)
    ext[:, :, :3] = np.eye(3)
    ext[:, :, 3] = rng.normal(size=(n, 3))
    intr = np.tile(np.array([[100.0, 0, 2], [0, 100.0, 2], [0, 0, 1]], np.float32), (n, 1, 1))
    return ext, intr


def _pose_geometry_case(name):
    """(gt ext, intr, pred ext, check(out, ref)) of one edge case."""
    if name == "coincident_gt":
        ext, intr, pred = _ring(6, 21)
        ext[0, :, 3] = ext[1, :, 3] = 0                  # both centres at the origin: t_01 = 0 exactly

        def check(out, ref):
            assert float(out["pair_errors"][0, 1]) == 90.0
        return ext, intr, pred, check
    if name == "coincident_pred":
        ext, intr, pred = _ring(6, 22)
        pred[2, :, 3] = pred[4, :, 3] = 0

        def check(out, ref):
            k = list(map(tuple, ref["pairs"].tolist())).index((2, 4))
            assert float(out["pair_errors"][k, 1]) == 90.0
        return ext, intr, pred, check
    if name == "antiparallel":
        ext, intr = _identity_cams(6, 23)
        pred = ext.copy()
        pred[:, :, 3] = -ext[:, :, 3]                     # every t_ij,pred = -t_ij,gt: e = 180, folded to 0

        def check(out, ref):
            e = out["pair_errors"].cpu().numpy()
            assert (e[:, 0] == 0).all() and np.abs(e[:, 1]).max() < 1e-9
            assert (out["auc"].cpu().numpy() == 1).all()
        return ext, intr, pred, check
    if name == "rotation_near_0_and_180":
        ext, intr, _ = _ring(5, 24)
        pred = ext.astype(np.float64)
        for v, deg in ((1, 179.9999), (3, 1e-4), (4, 180.0)):    # about each camera's own y axis: the centre stays
            R = rot_y(deg)
            pred[v, :, :3] = R @ pred[v, :, :3]
            pred[v, :, 3] = R @ pred[v, :, 3]
        pred = pred.astype(np.float32)

        def check(out, ref):
            rre = ref["pair_errors"][:, 0]
            assert rre.max() > 179.99 and (rre[rre > 1] > 100).any() and rre.min() < 1e-3
        return ext, intr, pred, check
    if name == "equal":
        ext, intr, _ = _ring(7, 25)
        return ext, intr, ext.copy(), None
    if name == "duplicate_consecutive":
        ext, intr = _identity_cams(6, 26)
        ext[3] = ext[2]
        rng = np.random.default_rng(126)
        pred = ext.copy()
        pred[:, :, 3] += rng.normal(0, 0.05, (6, 3)).astype(np.float32)
        pred[3] = pred[2]

        def check(out, ref):
            assert np.abs(out["rpe_errors"][2].cpu().numpy()).max() < 1e-6     # the repeated pose is a step of zero
            k = list(map(tuple, ref["pairs"].tolist())).index((2, 3))
            assert float(out["pair_errors"][k, 1]) == 90.0
        return ext, intr, pred, check
    if name == "three_views":
        ext, intr, pred = _ring(3, 27)
        return ext, intr, pred, None
    if name == "centre_overflow":
        ext, intr, pred = _ring(8, 28)
        ext[2] = _overflowing(ext[2])
        pred[5] = _overflowing(pred[5])

        def check(out, ref):
            assert list(ref["views"]) == [0, 1, 3, 4, 6, 7]
            assert not np.isin(out["pairs"].cpu().numpy(), [2, 5]).any()
        return ext, intr, pred, check
    raise KeyError(name)


POSE_EDGES = ["coincident_gt", "coincident_pred", "antiparallel", "rotation_near_0_and_180", "equal", "duplicate_consecutive",
              "three_views", "centre_overflow"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", POSE_EDGES)
def test_pose_geometry_edges_against_the_oracle(name):
    from omnivggt_official_b200 import OmniVGGT
    ext, intr, pred, check = _pose_geometry_case(name)
    n = len(ext)
    out = OmniVGGT.evaluate(_pred(n, 4, 4, extrinsic=_cuda(pred)[None]), extrinsics=_cuda(ext)[None],
                            intrinsics=_cuda(intr)[None])["pose"]
    ref = _check_pose(out, ext, intr, pred, atol=1e-12)
    if check is not None:
        check(out, ref)


# ------------------------------------------------------------------------------------------------------------------ GPU: depth
def _eval_depth(gt, pred, mask=None, views=None):
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = gt.shape
    kw = {} if mask is None else {"mask": _cuda(mask)[None]}
    return OmniVGGT.evaluate(_pred(S, H, W, depth=_cuda(pred)[None, ..., None]), depth=_cuda(gt)[None], views=views,
                             **kw)["depth"]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 5, 7), (1, 1, 3), (5, 17, 13), (2, 1, 1)], ids=str)
def test_depth_at_odd_shapes_against_the_oracle(shape):
    rng = np.random.default_rng(sum(shape))
    gt = rng.uniform(0.5, 8, shape).astype(np.float32)
    gt[rng.uniform(size=shape) < 0.1] = 0
    pred = (gt * rng.uniform(0.6, 1.6, shape) + 0.1).astype(np.float32)
    mask = rng.uniform(size=shape) > 0.1
    mask.reshape(-1)[0] = True
    gt.reshape(-1)[0] = 2.0
    _check_depth_dicts(_eval_depth(gt, pred, mask), EO.depth_metrics(gt, pred, mask))


@pytest.mark.gpu
def test_depth_delta_thresholds_are_strict():
    S, H, W = 3, 8, 8
    gt = np.full((S, H, W), 2.0, np.float32)
    gt[2, :4, :4] = 0.5                                   # a second power of two
    pred = gt.copy()                                      # most pixels exact: both medians 2, the scale exactly 1
    picks = iter([(0, 1, 1), (0, 3, 5), (1, 0, 0), (1, 7, 7), (1, 4, 2), (0, 6, 6), (2, 0, 0), (2, 1, 3), (2, 3, 1), (2, 2, 2),
                  (2, 0, 3), (2, 3, 3)])
    for t in (1.25, 1.5625, 1.953125):
        for _ in range(2):
            v, y, x = next(picks)
            g = gt[v, y, x]
            at = np.float32(t * g)
            assert at == t * float(g)                     # exactly on the threshold
            pred[v, y, x] = at
            v, y, x = next(picks)
            pred[v, y, x] = np.nextafter(np.float32(t * gt[v, y, x]), np.float32(0))
    out = _eval_depth(gt, pred)
    ref = EO.depth_metrics(gt, pred)
    assert float(out["scale"]) == 1.0 == ref["scale"]
    _check_depth_dicts(out, ref)
    n = S * H * W
    assert list(ref["delta_counts"]) == [n - 10, n - 6, n - 2]    # on a threshold: out; one ulp below: in


def _median_case(name):
    """(gt, pred, mask) [2, 4, 5] whose valid pixels exercise one median case."""
    gt = np.ones((2, 4, 5), np.float32)
    pred = np.ones((2, 4, 5), np.float32)
    mask = np.zeros((2, 4, 5), bool)
    rng = np.random.default_rng(len(name))
    flat = rng.permutation(40)

    def put(gvals, pvals):
        idx = flat[:len(gvals)]
        mask.reshape(-1)[idx] = True
        gt.reshape(-1)[idx] = gvals
        pred.reshape(-1)[idx] = pvals

    if name == "odd":
        put(rng.uniform(1, 5, 7), rng.uniform(1, 5, 7))
    elif name == "even":
        put(rng.uniform(1, 5, 8), rng.uniform(1, 5, 8))
    elif name == "one":
        put([3.0], [1.5])
    elif name == "all_equal":
        put(np.full(9, 2.5), np.full(9, 0.75))
    elif name == "ties_across_middle":
        put([1, 2, 3, 3, 3, 3, 5, 6], [0.5, 4, 4, 4, 4, 7, 8, 9])
    elif name == "ties_straddling":
        put([1, 2, 2, 3, 3, 4], [1, 1, 1, 2, 2, 2])
    elif name == "zero_pred":
        put(rng.uniform(1, 5, 9), [0, 0, 0, 0, 0, 1, 2, 3, 4])
    elif name == "negative_pred":
        put(rng.uniform(1, 5, 9), [-3, -2, -1, -1, -0.5, 0, 1, 2, 3])
    elif name == "negative_median":
        put(rng.uniform(1, 5, 8), [-3, -2, -2, -1, -1, 0.5, 1, 2])
    else:
        raise KeyError(name)
    return gt, pred, mask


MEDIANS = ["odd", "even", "one", "all_equal", "ties_across_middle", "ties_straddling", "zero_pred", "negative_pred",
           "negative_median"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", MEDIANS)
def test_depth_medians_and_signs_like_numpy(name):
    gt, pred, mask = _median_case(name)
    ref = EO.depth_metrics(gt, pred, mask)
    out = _eval_depth(gt, pred, mask)
    _check_depth_dicts(out, ref)
    if name in ("zero_pred", "negative_pred"):
        assert not np.isfinite(ref["abs_rel"]) or ref["scale"] <= 0


@pytest.mark.gpu
def test_depth_past_65535_views_against_the_oracle():
    S, H, W = 65537, 4, 4
    rng = np.random.default_rng(65537)
    gt = rng.uniform(0.5, 8, (S, H, W)).astype(np.float32)
    pred = (gt * rng.uniform(0.7, 1.5, gt.shape)).astype(np.float32)
    mask = rng.uniform(size=gt.shape) > 0.2
    mask[-1] = False                                      # the last view without pixels: NaN
    views = [v for v in range(S) if v % 7]
    out = _eval_depth(gt, pred, mask, views)
    ref = EO.depth_metrics(gt, pred, mask, views)
    _check_depth_dicts(out, ref)
    assert int(out["view_pixels"][65536]) == 0 and int(out["view_pixels"][65535]) > 0


@pytest.mark.gpu
def test_depth_past_2gib_of_selection_columns_against_the_oracle():
    """S H W > 2^29: the predicted depths' selection column starts past 2 GiB of the workspace."""
    S, H, W = 33, 4096, 3985
    assert S * H * W > 2 ** 29
    gt = np.empty((S, H, W), np.float32)
    pred = np.empty((S, H, W), np.float32)
    for v in range(S):                                    # view by view, to keep the host's peak down
        rng = np.random.default_rng(1000 + v)
        gt[v] = rng.uniform(0.5, 20, (H, W))
        gt[v, :, :: 5 + v % 3] = 0                       # invalid columns
        pred[v] = gt[v] * rng.uniform(0.5, 2.0, (H, W)) + 0.01
    out = _eval_depth(gt, pred)
    ref = EO.depth_metrics(gt, pred, chunk=1)
    _check_depth_dicts(out, ref)


# ------------------------------------------------------------------------------------------------------------------ GPU: points
def _eval_points(ext, intr, depth, pts, pred_ext, views=None, depth_arg=None):
    from omnivggt_official_b200 import OmniVGGT
    S, H, W = depth.shape
    pred = _pred(S, H, W, extrinsic=_cuda(pred_ext)[None], depth=_cuda(depth)[None], world_points_from_depth=_cuda(pts)[None])
    return OmniVGGT.evaluate(pred, extrinsics=_cuda(ext)[None], intrinsics=_cuda(intr)[None],
                             depth=_cuda(depth)[None] if depth_arg is None else depth_arg, views=views)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 5, 7), (6, 5, 7), (5, 5, 7), (3, 9, 13)], ids=str)
@pytest.mark.parametrize("offset", [False, True], ids=["dense", "odd_offset_depth"])
def test_points_at_odd_pixel_counts_against_the_oracle(shape, offset):
    S, H, W = shape
    ext, intr, depth, pts, pred_ext = _points_case(S, H, W, seed=S * H * W)
    arg = None
    if offset:
        buf = torch.zeros(depth.size + 3, device="cuda")
        buf[3:] = _cuda(depth).reshape(-1)
        arg = buf[3:].view(1, S, H, W)
        assert arg.data_ptr() % 16 != 0
    out = _eval_points(ext, intr, depth, pts, pred_ext, depth_arg=arg)
    _check_points(out["points"], ext, intr, depth, pts)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(6, 1, 9), (6, 2, 9), (6, 9, 1), (6, 9, 2), (6, 2, 2)], ids=str)
def test_points_without_normals_give_nan_nc(shape):
    S, H, W = shape
    ext, intr, depth, pts, pred_ext = _points_case(S, H, W, seed=31)
    depth, pts = _full_frame(S, H, W, ext, intr, seed=31)
    out = _eval_points(ext, intr, depth, pts, pred_ext)["points"]
    for k in ("nc_acc", "nc_comp", "nc"):
        assert np.isnan(float(out[k])), k
    _check_points(out, ext, intr, depth, pts)


def _full_frame(S, H, W, ext, intr, seed):
    """Depth of a sphere of radius 2 seen from about 3 away (at a focal length of 0.9 W every pixel sees it), and a noisy
    similarity of its points."""
    from test_evaluate import sim3_of
    rng = np.random.default_rng(seed)
    depth = np.empty((S, H, W), np.float32)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    for s in range(S):
        E = ext[s].astype(np.float64)
        R, c = E[:, :3], -E[:, :3].T @ E[:, 3]
        K = intr[s].astype(np.float64)
        d = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1) @ R
        a2, b = (d * d).sum(-1), 2 * (d @ c)
        disc = b * b - 4 * a2 * (c @ c - 4.0)
        depth[s] = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a2), 0.0)
    sc, R, t = sim3_of(rng)
    pts = (sc * EO.unproject(depth, ext, intr) @ R.T + t + rng.normal(0, 0.002, depth.shape + (3,))).astype(np.float32)
    pts[depth == 0] = np.nan
    return depth, pts


@pytest.mark.gpu
def test_points_with_border_holes_and_a_views_subset():
    S, H, W = 6, 24, 32
    ext, intr, _, _, pred_ext = _points_case(S, H, W, seed=41)
    depth, pts = _full_frame(S, H, W, ext, intr, seed=41)
    assert (depth > 0).all()
    depth[0, 0, :] = 0                                    # holes along every border, in the ground truth ...
    depth[1, :, -1] = 0
    depth[2, -3:, :] = 0
    pts[3, :, :2] = np.nan                                # ... and in the prediction
    pts[4, 0, 0] = pts[4, -1, -1] = np.nan
    depth[5, 10:14, 0:6] = 0
    views = [0, 1, 2, 3, 4]
    out = _eval_points(ext, intr, depth, pts, pred_ext, views=views)["points"]
    _check_points(out, ext, intr, depth, pts, views)


@pytest.mark.gpu
def test_points_with_one_kept_pixel_per_view():
    S, H, W = 7, 10, 10
    ext, intr, _, _, pred_ext = _points_case(S, H, W, seed=43)
    depth, pts = _full_frame(S, H, W, ext, intr, seed=43)
    at = [(0, 0), (H - 1, W - 1), (0, W - 1), (H - 1, 0), (5, 0), (0, 4), (6, 5)]
    keep = np.zeros_like(depth, bool)
    for s, (y, x) in enumerate(at):
        keep[s, y, x] = True
    depth[~keep] = 0
    out = _eval_points(ext, intr, depth, pts, pred_ext)["points"]
    assert int(out["pixels"]) == S and np.isnan(float(out["nc"]))
    _check_points(out, ext, intr, depth, pts)
