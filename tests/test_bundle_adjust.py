"""OmniVGGT.bundle_adjust (scene.bundle_adjust, libovg ovg_bundle_adjust): the numpy oracle against central differences,
scipy.optimize.least_squares and the truth on the host; the device against the oracle, step for step, on the H100."""
import numpy as np
import pytest
import torch

from oracle import ba_oracle as BO
from ovg_support import install


# ------------------------------------------------------------------------------------------------------------------ scenes
def synthetic(V=5, n=400, seed=0, noise=0.3, gauge_at_truth=False):
    """A seeded scene of V cameras on an arc looking at n points: (inputs of ovg_bundle_adjust as numpy, truth).
    Observations are the truth's projections plus ``noise`` pixels; the cameras handed in are the truth perturbed by 0.01 rad,
    1 % of the translation and 2 % of the focal length, the points by 1 %.  With ``gauge_at_truth`` view 0's pose and view
    1's held translation coordinate are the truth's and the noise is zero."""
    rng = np.random.default_rng(seed)
    Pt = rng.uniform(-1.0, 1.0, (n, 3))
    ext = np.zeros((V, 3, 4))
    intr = np.zeros((V, 3, 3))
    for v in range(V):
        a = 0.6 * (v - (V - 1) / 2)
        R = BO.exp_so3(np.array([0.0, a, 0.0]))
        C = np.array([2.5 * np.sin(a), 0.5 * rng.standard_normal(), -2.5 * np.cos(a)])
        ext[v] = np.c_[R, -R @ C]
        f = 200.0 * (1 + 0.05 * rng.standard_normal())
        intr[v] = [[f, 0, 100.0], [0, f * (1 + 0.01 * rng.standard_normal()), 90.0], [0, 0, 1]]
    ext32, intr32 = ext.astype(np.float32), intr.astype(np.float32)        # what the call is handed
    # the truth: the handed cameras moved by the perturbation, so the left increments reach it exactly
    Et, Kt = ext32.astype(np.float64), intr32.astype(np.float64)
    for v in range(V):
        Et[v, :, :3] = BO.exp_so3(0.01 * rng.standard_normal(3) / np.sqrt(3)) @ Et[v, :, :3]
        Et[v, :, 3] *= 1 + 0.01 * rng.standard_normal(3)
        Kt[v, 0, 0] *= 1 + 0.02 * rng.standard_normal()
        Kt[v, 1, 1] *= 1 + 0.02 * rng.standard_normal()
    if gauge_at_truth:
        k = BO.Problem(Pt, np.arange(n + 1), np.zeros(n, np.int64), np.zeros((n, 2)), ext32, intr32).k
        Et[0] = ext32[0]
        Et[1, k, 3] = ext32[1, k, 3]
        noise = 0.0
    views, offsets = [], [0]
    for p in range(n):
        vs = np.sort(rng.choice(V, size=int(rng.integers(2, V + 1)), replace=False))
        views.append(vs)
        offsets.append(offsets[-1] + len(vs))
    view = np.concatenate(views).astype(np.int32)
    offsets = np.array(offsets, np.int64)
    track = np.repeat(np.arange(n), np.diff(offsets))
    _, r, behind = BO.reproject(Et[view], Kt[view], Pt[track], np.zeros((len(view), 2)))
    assert not behind.any()
    obs = r + noise * rng.standard_normal(r.shape)
    P0 = Pt * (1 + 0.01 * rng.standard_normal(Pt.shape))
    return dict(points=P0, offsets=offsets, view=view, obs=obs, ext=ext32, intr=intr32), (Pt, Et, Kt)


def scipy_cost(inp, refine_focal, loss, loss_scale, start=None):
    """The same problem solved by scipy.optimize.least_squares over the free parameters (rotation vectors of the left
    increments, translations, focal lengths, points of the refined tracks); returns its final cost.  scipy applies the loss to
    each residual, so with a robust loss its residual of an observation is the distance |r_o|, whose square is the s of
    rho(s).  ``start``: (extrinsic, intrinsic, points) to start from instead of the inputs."""
    from scipy.optimize import least_squares
    pr = BO.Problem(inp["points"], inp["offsets"], inp["view"], inp["obs"], inp["ext"], inp["intr"], refine_focal, loss,
                    loss_scale)
    if start is not None:
        pr.E0, pr.K0, pr.P0 = (np.array(a, np.float64) for a in start)
    V, mask, io = pr.V, pr.mask, pr.io
    free = mask.ravel() != 0
    inc = np.flatnonzero(pr.incl)

    def unpack(z):
        c = np.zeros(V * BO.NP)
        c[free] = z[:free.sum()]
        c = c.reshape(V, BO.NP)
        E, K, P = pr.E0.copy(), pr.K0.copy(), pr.P0.copy()
        E[:, :, :3] = BO.exp_so3(c[:, :3]) @ pr.E0[:, :, :3]
        E[:, :, 3] += c[:, 3:6]
        K[:, 0, 0] += c[:, 6]
        K[:, 1, 1] += c[:, 7]
        P[inc] += z[free.sum():].reshape(-1, 3)
        return E, K, P

    def fun(z):
        E, K, P = unpack(z)
        _, r, _ = BO.reproject(E[pr.view[io]], K[pr.view[io]], P[pr.track[io]], pr.obs[io])
        return r.ravel() if loss == "trivial" else np.sqrt((r * r).sum(1))

    z0 = np.zeros(free.sum() + 3 * len(inc))
    sol = least_squares(fun, z0, method="trf", loss="linear" if loss == "trivial" else "cauchy", f_scale=loss_scale,
                        ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=400)
    return sol.cost


# ------------------------------------------------------------------------------------------------------------------ oracle
def test_oracle_jacobian_matches_central_differences():
    inp, _ = synthetic(V=4, n=30, seed=1)
    pr = BO.Problem(inp["points"], inp["offsets"], inp["view"], inp["obs"], inp["ext"], inp["intr"])
    E, K, P = pr.E0[pr.view], pr.K0[pr.view], pr.P0[pr.track]
    mask = np.ones((len(pr.view), BO.NP))
    r, jc, jp = BO.jacobians(E, K, P, pr.obs, mask)
    h = 1e-6
    for i in range(BO.NP):
        d = np.zeros(BO.NP)
        d[i] = h
        res = []
        for s in (1, -1):
            E2, K2 = E.copy(), K.copy()
            E2[:, :, :3] = BO.exp_so3(s * d[:3]) @ E[:, :, :3]
            E2[:, :, 3] += s * d[3:6]
            K2[:, 0, 0] += s * d[6]
            K2[:, 1, 1] += s * d[7]
            res.append(BO.reproject(E2, K2, P, pr.obs)[1])
        num = (res[0] - res[1]) / (2 * h)
        assert np.allclose(num, jc[:, :, i], rtol=1e-6, atol=1e-6 * np.abs(jc).max()), i
    for a in range(3):
        d = np.zeros(3)
        d[a] = h
        num = (BO.reproject(E, K, P + d, pr.obs)[1] - BO.reproject(E, K, P - d, pr.obs)[1]) / (2 * h)
        assert np.allclose(num, jp[:, :, a], rtol=1e-6, atol=1e-6 * np.abs(jp).max()), a


@pytest.mark.parametrize("seed,V,n,refine_focal,loss,scale", [(4, 4, 300, False, "trivial", 1.0), (9, 6, 400, True, "trivial", 1.0),
                                                              (7, 5, 250, True, "trivial", 1.0), (7, 5, 250, True, "cauchy", 2.0)])
def test_oracle_matches_scipy_and_direct_solves(seed, V, n, refine_focal, loss, scale):
    inp, _ = synthetic(V=V, n=n, seed=seed)
    got = BO.bundle_adjust(inp["points"], inp["offsets"], inp["view"], inp["obs"], inp["ext"], inp["intr"], iterations=100,
                           refine_focal=refine_focal, loss=loss, loss_scale=scale, record=True)
    assert got["status"] == 0 and got["cost"][1] < got["cost"][0]
    assert np.all(np.diff(got["trace"]) <= 0)
    if loss == "trivial":
        want = scipy_cost(inp, refine_focal, loss, scale)
        assert abs(got["cost"][1] - want) <= 1e-8 * want, (got["cost"][1], want)
    else:
        # scipy's trust-region path with a robust loss and finite-difference Jacobians does not converge from the perturbed
        # start in a usable time (over 10 minutes at 1000 evaluations on this 250-track scene), so the independent solve from
        # the same start is the trivial-loss cases above.  Here scipy starts at the oracle's minimum and must find nothing
        # lower: the oracle stopped at a minimum of the robust cost, not only where its own IRLS rules say so.
        want = scipy_cost(inp, refine_focal, loss, scale, start=(got["extrinsic"], got["intrinsic"], got["points"]))
        assert want >= got["cost"][1] * (1 - 1e-8), (got["cost"][1], want)
    for x, direct in got["solves"]:
        assert np.linalg.norm(x - direct) <= 1e-8 * np.linalg.norm(direct)


def test_oracle_converges_to_the_truth_without_noise():
    inp, (Pt, Et, Kt) = synthetic(V=5, n=300, seed=5, gauge_at_truth=True)
    got = BO.bundle_adjust(inp["points"], inp["offsets"], inp["view"], inp["obs"], inp["ext"], inp["intr"])
    assert got["status"] == 0
    assert np.abs(got["extrinsic"] - Et).max() <= 1e-9
    assert np.abs(got["intrinsic"] - Kt).max() <= 1e-9 * 200
    assert np.abs(got["points"] - Pt).max() <= 1e-9


# ------------------------------------------------------------------------------------------------------------------ dry runs
@pytest.fixture()
def dry(monkeypatch):
    return install(monkeypatch, workspace_bytes=256)


def _tracks_dict(V=3, n=4, m=9):
    return {"points": torch.zeros(n, 3, dtype=torch.float64), "colors": torch.zeros(n, 3, dtype=torch.uint8),
            "error": torch.zeros(n, dtype=torch.float64), "offsets": torch.zeros(n + 1, dtype=torch.int64),
            "view": torch.zeros(m, dtype=torch.int32), "xy": torch.zeros(m, 2, dtype=torch.int64),
            "point2d": torch.zeros(m, dtype=torch.int32), "view_offsets": torch.zeros(V + 1, dtype=torch.int64),
            "view_track": torch.zeros(m, dtype=torch.int32), "view_xy": torch.zeros(m, 2, dtype=torch.int64),
            "extrinsic": torch.zeros(V, 3, 4), "intrinsic": torch.zeros(V, 3, 3)}


def test_dry_run_one_call_no_host_read(dry):
    from omnivggt_official_b200 import OmniVGGT
    tr = _tracks_dict()
    out = OmniVGGT.bundle_adjust(tr, iterations=7, refine_focal=False, loss="cauchy", loss_scale=2.0)
    assert dry.names() == ["ovg_ba_workspace_bytes", "ovg_bundle_adjust"]
    assert dry.args("ovg_ba_workspace_bytes")[0] == (3, 4, 9)
    a = dry.args("ovg_bundle_adjust")[0]
    assert a[6:13] == (3, 4, 9, 7, 0, 1, 2.0) and a[-2] is None
    assert len(dry.reads) == 0
    assert set(out) == set(tr) | {"ba"}
    for k in ("colors", "offsets", "view", "xy", "point2d", "view_offsets", "view_track", "view_xy"):
        assert out[k] is tr[k]
    assert out["points"].dtype == out["extrinsic"].dtype == out["intrinsic"].dtype == torch.float64
    assert set(out["ba"]) == {"cost", "steps", "accepted", "pcg_iterations", "status"}
    assert out["ba"]["status"].dtype == torch.int32 and out["ba"]["steps"].dtype == torch.int64


def test_errors_before_any_library_call(dry):
    from omnivggt_official_b200 import OmniVGGT
    tr = _tracks_dict()
    for kw, match in ((dict(iterations=0), "iterations"), (dict(iterations=2.0), "iterations"),
                      (dict(iterations=True), "iterations"), (dict(loss="huber"), "loss"), (dict(loss_scale=0.0), "loss_scale"),
                      (dict(loss_scale=float("nan")), "loss_scale"), (dict(loss_scale=float("inf")), "loss_scale"),
                      (dict(loss_scale="1"), "loss_scale"), (dict(iterations=2 ** 31), "iterations")):
        with pytest.raises(ValueError, match=match):
            OmniVGGT.bundle_adjust(tr, **kw)
    with pytest.raises(ValueError, match="views"):
        OmniVGGT.bundle_adjust(_tracks_dict(V=1))
    for k, bad in (("points", torch.zeros(4, 3)), ("view", torch.zeros(9, dtype=torch.int64)), ("offsets", torch.zeros(4, dtype=torch.int64)),
                   ("extrinsic", torch.zeros(3, 3, 4, dtype=torch.float64)), ("xy", torch.zeros(8, 2, dtype=torch.int64))):
        with pytest.raises(ValueError, match=k):
            OmniVGGT.bundle_adjust({**tr, k: bad})
    with pytest.raises(ValueError, match="tracks"):
        OmniVGGT.bundle_adjust({k: v for k, v in tr.items() if k != "view_xy"})
    with pytest.raises(ValueError, match="device"):
        OmniVGGT.bundle_adjust({**tr, "points": torch.zeros(4, 3, dtype=torch.float64, device="meta")})
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
def _device(inp, **kw):
    from omnivggt_official_b200 import ops
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)
    return ops.bundle_adjust(t(inp["points"], torch.float64), t(inp["offsets"], torch.int64), t(inp["view"], torch.int32),
                             t(inp["obs"], torch.float64), t(inp["ext"], torch.float32), t(inp["intr"], torch.float32),
                             trace=True, **kw)


def _oracle(inp, **kw):
    return BO.bundle_adjust(inp["points"], inp["offsets"], inp["view"], inp["obs"], inp["ext"], inp["intr"], **kw)


RTOL = 1e-7                   # final points and cameras, device against oracle, relative to each array's largest value


def _assert_matches(got, want, iterations):
    pts, ext, intr, err, cost, stats, trace = (t.cpu().numpy() for t in got)
    steps, acc, pcg, status = stats.tolist()
    assert (steps, acc, status) == (want["steps"], want["accepted"], want["status"]), (stats, want["steps"], want["accepted"],
                                                                                      want["status"])
    assert abs(pcg - want["pcg_iterations"]) <= max(2, 0.02 * want["pcg_iterations"]), (pcg, want["pcg_iterations"])
    np.testing.assert_allclose(trace[:steps], want["trace"], rtol=1e-9, atol=0)
    assert np.isnan(trace[steps:]).all()
    np.testing.assert_allclose(cost, want["cost"], rtol=1e-9, atol=0)
    for a, b in ((pts, want["points"]), (ext, want["extrinsic"]), (intr, want["intrinsic"])):
        assert np.abs(a - b).max() <= RTOL * np.abs(b).max(), np.abs(a - b).max() / np.abs(b).max()
    fin = np.isfinite(want["error"])
    assert np.array_equal(np.isfinite(err), fin)
    np.testing.assert_allclose(err[fin], want["error"][fin], rtol=1e-6, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("loss,scale", [("trivial", 1.0), ("cauchy", 0.7)])
@pytest.mark.parametrize("seed,V,n,refine_focal", [(2, 3, 300, True), (3, 6, 2000, True), (4, 4, 800, False), (6, 12, 5000, True)])
def test_device_matches_oracle_step_for_step(seed, V, n, refine_focal, loss, scale):
    inp, _ = synthetic(V=V, n=n, seed=seed)
    kw = dict(iterations=50, refine_focal=refine_focal, loss=loss, loss_scale=scale)
    _assert_matches(_device(inp, **kw), _oracle(inp, **kw), 50)


@pytest.mark.gpu
def test_device_converges_to_the_truth_and_holds_the_gauge():
    inp, (Pt, Et, Kt) = synthetic(V=5, n=300, seed=5, gauge_at_truth=True)
    pts, ext, intr, err, cost, stats, _ = (t.cpu().numpy() for t in _device(inp, iterations=100, refine_focal=True,
                                                                             loss="trivial", loss_scale=1.0))
    assert stats[3] == 0
    assert np.abs(ext - Et).max() <= 1e-9 and np.abs(intr - Kt).max() <= 1e-9 * 200 and np.abs(pts - Pt).max() <= 1e-9
    k = BO.Problem(inp["points"], inp["offsets"], inp["view"], inp["obs"], inp["ext"], inp["intr"]).k
    e32 = inp["ext"].astype(np.float64)
    assert ext[0].tobytes() == e32[0].tobytes() and ext[1, k, 3].tobytes() == e32[1, k, 3].tobytes()


@pytest.mark.gpu
def test_repeatable_poison_free_and_excluded_tracks_held():
    from test_poison_gpu import check_case
    inp, _ = synthetic(V=4, n=600, seed=8)
    inp["points"][:5, 2] = -50.0                      # behind every camera: held
    kw = dict(iterations=30, refine_focal=True, loss="cauchy", loss_scale=1.0)
    a, b = _device(inp, **kw), _device(inp, **kw)
    for x, y in zip(a, b):
        assert torch.equal(x.view(-1).view(torch.uint8), y.view(-1).view(torch.uint8))
    assert torch.equal(a[0][:5].cpu(), torch.from_numpy(inp["points"][:5]))
    assert torch.isinf(a[3][:5]).all()
    check_case("bundle_adjust", lambda P: _device(inp, **kw), finite=())


def _surface_tracks(S, pairs, H=96, W=128, seed=0, perturb=True):
    """tracks() on a surface-like scene (tools/tracks_bench.py's at a smaller size) with the cameras handed to it perturbed:
    rotation 0.01 rad, translation 1 %, focal 2 %."""
    from omnivggt_official_b200 import OmniVGGT
    from oracle.make_golden_matches import surface_views
    from test_tracks import _scene
    pred = {k: v.cuda() for k, v in _scene(S, H, W, seed).items()}
    pred["world_points_from_depth"] = torch.from_numpy(surface_views(S, H, W, seed))[None].cuda()
    truth = _surface_cameras(S, H, W)
    ext, intr = (torch.from_numpy(a).float().cuda() for a in truth)
    if perturb:
        rng = np.random.default_rng(seed + 1)
        e, k = truth[0].copy(), truth[1].copy()
        for v in range(S):
            e[v, :, :3] = BO.exp_so3(0.01 * rng.standard_normal(3) / np.sqrt(3)) @ e[v, :, :3]
            e[v, :, 3] *= 1 + 0.01 * rng.standard_normal(3)
            k[v, :2, :2] *= 1 + 0.02 * rng.standard_normal()
        ext, intr = torch.from_numpy(e).float().cuda(), torch.from_numpy(k).float().cuda()
    pred["extrinsic"], pred["intrinsic"] = ext[None], intr[None]
    return OmniVGGT.tracks(pred, pairs), pred, truth


def _surface_cameras(S, H, W):
    """The cameras surface_views unprojects through: f = 0.9 W, principal point (W/2 - 1.5 s, H/2) in the reference's
    convention, and a rotation of 0.05 s about y with a 0.02 s shift in z (world-to-camera)."""
    ext = np.zeros((S, 3, 4))
    intr = np.zeros((S, 3, 3))
    for s in range(S):
        a = 0.05 * s
        Rcw = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])   # camera -> world
        ext[s] = np.c_[Rcw.T, -Rcw.T @ np.array([0, 0, 0.02 * s])]
        intr[s] = [[0.9 * W, 0, W / 2 - 1.5 * s], [0, 0.9 * W, H / 2], [0, 0, 1]]
    return ext, intr


def _ranking_pairs(S):
    import sys
    import os
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from tracks_bench import ranking_pairs
    return ranking_pairs(S)


@pytest.mark.gpu
@pytest.mark.parametrize("S,ranking,loss,refine_focal", [(8, False, "trivial", True), (8, False, "cauchy", False),
                                                         (24, True, "trivial", True), (24, True, "cauchy", True)])
def test_surface_scenes_match_oracle(S, ranking, loss, refine_focal):
    from omnivggt_official_b200 import ops
    tr, _, _ = _surface_tracks(S, _ranking_pairs(S) if ranking else None)
    kw = dict(iterations=15, refine_focal=refine_focal, loss=loss, loss_scale=1.0)
    obs = tr["xy"].double() + 0.5
    got = ops.bundle_adjust(tr["points"], tr["offsets"], tr["view"], obs, tr["extrinsic"].contiguous(),
                            tr["intrinsic"].contiguous(), trace=True, **kw)
    want = BO.bundle_adjust(*(t.cpu().numpy() for t in (tr["points"], tr["offsets"], tr["view"], obs, tr["extrinsic"],
                                                       tr["intrinsic"])), **kw)
    _assert_matches(got, want, 15)


def _bowl_scene(S=6, H=120, W=160, seed=0, pose=1.0, focal=1.0):
    """Predictions whose point maps all lie on one surface, z = 2.5 + 0.3 (x^2 + y^2), ray-cast through true cameras on an
    arc 2 units from the bowl's bottom, 0.15 rad apart; the cameras handed in are the truth with views 1.. perturbed (``pose``
    times 0.01 rad and 1 % of the translation, ``focal`` times 2 % of the focal length) and view 1's translation kept, so the
    gauge is the truth's.  Returns (predictions, true extrinsic, intrinsic)."""
    rng = np.random.default_rng(seed)
    Et, Kt = np.zeros((S, 3, 4)), np.zeros((S, 3, 3))
    pts = np.zeros((S, H, W, 3))
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    for s in range(S):
        a = 0.15 * (s - (S - 1) / 2)
        R = BO.exp_so3(np.array([0.0, a, 0.0]))
        C = np.array([2.0 * np.sin(a), 0.05 * s, 2.5 - 2.0 * np.cos(a)])
        Et[s] = np.c_[R, -R @ C]
        f = 0.9 * W
        Kt[s] = [[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]]
        d = np.stack([(u - W / 2) / f, (v - H / 2) / f, np.ones_like(u)], -1) @ R      # world ray directions (R^T d)
        qa = 0.3 * (d[..., 0] ** 2 + d[..., 1] ** 2)
        qb = 0.6 * (C[0] * d[..., 0] + C[1] * d[..., 1]) - d[..., 2]
        qc = 2.5 + 0.3 * (C[0] ** 2 + C[1] ** 2) - C[2]
        lam = np.where(qa > 1e-12, (-qb - np.sqrt(np.maximum(qb * qb - 4 * qa * qc, 0))) / (2 * np.maximum(qa, 1e-12)), -qc / qb)
        pts[s] = C + lam[..., None] * d
    E, K = Et.copy(), Kt.copy()
    for s in range(1, S):
        E[s, :, :3] = BO.exp_so3(pose * 0.01 * rng.standard_normal(3) / np.sqrt(3)) @ E[s, :, :3]
        if s > 1:
            E[s, :, 3] *= 1 + pose * 0.01 * rng.standard_normal(3)
        K[s, :2, :2] *= 1 + focal * 0.02 * rng.standard_normal()
    g = torch.Generator().manual_seed(seed)
    pred = {"images": torch.rand(1, S, 3, H, W, generator=g), "world_points_from_depth": torch.from_numpy(pts).float()[None],
            "depth_conf": 1.0 + torch.rand(1, S, H, W, generator=g), "extrinsic": torch.from_numpy(E).float()[None],
            "intrinsic": torch.from_numpy(K).float()[None]}
    return {k: t.cuda() for k, t in pred.items()}, Et, Kt


@pytest.mark.gpu
def test_end_to_end_export(tmp_path):
    """tracks -> bundle_adjust -> write_colmap: the cost and the mean track error go down and the written model holds the
    refined doubles; with every track held (status 3) the error is tracks' own, bit for bit."""
    from omnivggt_official_b200 import OmniVGGT
    from omnivggt_official_b200.colmap import write_colmap
    from oracle import tracks_oracle as TO
    pred, Et, Kt = _bowl_scene()
    tr = OmniVGGT.tracks(pred, conf_percent=0.0)
    out = OmniVGGT.bundle_adjust(tr)
    cost = out["ba"]["cost"].cpu().numpy()
    assert cost[1] <= cost[0] and int(out["ba"]["status"]) in (0, 1)
    fin = torch.isfinite(tr["error"])
    assert out["error"][fin].mean() < tr["error"][fin].mean()
    folder = write_colmap(str(tmp_path), pred, out, images=False)
    cams, _, pts = TO.read_model(folder, True)
    assert np.array_equal(np.array([p[1] for p in pts]), out["points"].cpu().numpy())
    assert np.array_equal(np.array([p[3] for p in pts]), out["error"].cpu().numpy())
    assert [c[4][:2] for c in cams] == out["intrinsic"][:, [0, 1], [0, 1]].cpu().tolist()
    one = OmniVGGT.tracks(pred, [], min_views=1)
    held = OmniVGGT.bundle_adjust(one)
    assert int(held["ba"]["status"]) == 3 and int(held["ba"]["steps"]) == 0
    assert held["error"].cpu().numpy().tobytes() == one["error"].cpu().numpy().tobytes()
    assert torch.equal(held["points"], one["points"])


@pytest.mark.gpu
def test_tracks_built_poses_move_towards_the_truth():
    """On tracks() of the bowl scene with the poses perturbed by 0.05 rad and 5 % of the translation and the focal lengths
    exact, refining the poses brings every camera within 0.05 of the truth (largest entry of [R | t]) from 0.067, and two
    different perturbations reach the same cameras.  The nearest-neighbour matches of grid-sampled point maps put the
    minimum about 0.03-0.05 from the truth; with the focal lengths refined the minimum on this scene is about 0.2 away
    (INTEGRATION.md, "Bundle adjustment", limits), so the focal lengths are held here."""
    from omnivggt_official_b200 import OmniVGGT
    ext = []
    for pose in (5.0, 1.0):
        pred, Et, _ = _bowl_scene(pose=pose, focal=0.0)
        tr = OmniVGGT.tracks(pred, conf_percent=0.0)
        out = OmniVGGT.bundle_adjust(tr, refine_focal=False)
        before = np.abs(tr["extrinsic"].double().cpu().numpy() - Et).max()
        after = np.abs(out["extrinsic"].cpu().numpy() - Et).max()
        print(f"pose perturbation x{pose}: camera error {before:.4f} -> {after:.4f}")
        if pose == 5.0:
            assert after < 0.05 < before, (before, after)
        ext.append(out["extrinsic"].cpu().numpy())
    assert np.abs(ext[0] - ext[1]).max() <= 1e-4


@pytest.mark.gpu
def test_reconstruct_tracks_bundle_adjust():
    from test_model_gpu import model
    from oracle.synth import make_inputs
    from omnivggt_official_b200.geometry import compute_ranking
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 10, 56, 56, seed=63).items()}
    rec = m.reconstruct(**inp, chunk=6, overlap=2)
    e = torch.eye(4, device="cuda", dtype=torch.float64).repeat(10, 1, 1)
    e[:, :3] = rec["extrinsic"][0].double()
    ranking, _ = compute_ranking(e, k=4)
    pairs = [(i, int(r)) for i, row in enumerate(ranking.cpu().tolist()) for r in row if r != i]
    tr = m.tracks(rec, pairs, conf_percent=25.0)
    out = m.bundle_adjust(tr, iterations=20)
    cost = out["ba"]["cost"].cpu().numpy()
    assert cost[1] <= cost[0]
