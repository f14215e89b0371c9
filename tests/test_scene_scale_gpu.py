"""Scene functions at long-capture view counts: bundle adjustment (csrc/ba.cuh) up to its 256-view limit, tracks and the fused
mesh at 64-96 views, and reconstruct -> tracks -> bundle_adjust / fused_mesh at 48 views.
CPU: the many-view scene generator's contract, and the numpy oracle on every bundle-adjustment case.
GPU: the device against the oracles: bundle adjustment step for step, tracks and the fused mesh bit for bit.

Which ba_pcg_kernel paths the view count selects (BA_PCG_THREADS = 256, BA_VIEW_SMEM = 104 doubles per view):
  owners       thread v owns view v: V > 32 puts owners in warps 1-7 and feeds their values into the block sums;
  grid         per_sm x SMs CTAs from the occupancy query at 832 V bytes of dynamic shared memory: one CTA per SM at V = 256;
  pass 2       V x BA_PCG_CHUNKS (view, chunk) items, one per warp, strided by the grid's warps: a warp takes several once the
               items outnumber the warps (V >~ 100);
  pass 1 and   tracks strided by the grid's threads: a thread takes several once there are more tracks than threads (about
  back-subst.  34 k at V = 256);
  edge views   a view without observations, or seen only by held tracks (its blocks are zero but for the damping); the last
               view, whose gather writes view_off[V]."""
import functools

import numpy as np
import pytest
import torch

from oracle import ba_oracle as BO
from test_bundle_adjust import _assert_matches, _device, _oracle, _ranking_pairs, _surface_tracks, max_rel_diff


# ------------------------------------------------------------------------------------------------------------------ scenes
def helix_scene(V, n, seed=0, views=(3, 8), unobserved=(), held=(), held_views=(), noise=0.3, distance=4.0):
    """A seeded scene of V cameras on a helix of T ~ sqrt(V / 4) turns around a column of n points: (inputs of
    ovg_bundle_adjust as numpy, truth, held).  Camera v sits at angle 2 pi (v mod P) / P of turn v // P (P views a turn),
    (P at least 8), ``distance`` (> 0.8) from the axis and looking at it, so every point (within 0.8 of the axis) is in front
    of every camera.  Track p is anchored at a view c (views in order for the first tracks, so every observed view has one, then at random) and seen
    by ``views`` (a range, inclusive) of its neighbours: the views at the next angles of c's turn, and of the turn above
    for half the tracks of four views or more.  ``unobserved`` views are never seen.  The perturbation is synthetic()'s:
    observations are the truth's projections plus ``noise`` pixels; the cameras handed in are the truth perturbed by 0.01
    rad, 1 % of the translation and 2 % of the focal length, the points by 1 %.  Tracks in ``held``, and every track that
    sees a view of ``held_views``, start 1 unit behind their first camera, so the adjuster holds them; ``held`` [n] marks
    them."""
    rng = np.random.default_rng(seed)
    T = max(1, int(round(np.sqrt(V / 4))))
    P = max(-(-V // T), 8)                          # at most 45 degrees between neighbours: no opposite-facing pair
    ext, intr = np.zeros((V, 3, 4)), np.zeros((V, 3, 3))
    for v in range(V):
        a = 2 * np.pi * (v % P) / P
        R = BO.exp_so3(np.array([0.02 * rng.standard_normal(), a, 0.02 * rng.standard_normal()]))   # no zero entries
        C = np.array([distance * np.sin(a), 0.5 * (v / P - T / 2), -distance * np.cos(a)])
        ext[v] = np.c_[R, -R @ C]
        f = 200.0 * (1 + 0.05 * rng.standard_normal())
        intr[v] = [[f, 0, 100.0], [0, f * (1 + 0.01 * rng.standard_normal()), 90.0], [0, 0, 1]]
    ext32, intr32 = ext.astype(np.float32), intr.astype(np.float32)
    Et, Kt = ext32.astype(np.float64), intr32.astype(np.float64)
    for v in range(V):
        Et[v, :, :3] = BO.exp_so3(0.01 * rng.standard_normal(3) / np.sqrt(3)) @ Et[v, :, :3]
        Et[v, :, 3] *= 1 + 0.01 * rng.standard_normal(3)
        Kt[v, 0, 0] *= 1 + 0.02 * rng.standard_normal()
        Kt[v, 1, 1] *= 1 + 0.02 * rng.standard_normal()
    ok = np.ones(V, bool)
    ok[list(unobserved)] = False
    anchors = np.flatnonzero(ok)
    lists, Pt = [], np.zeros((n, 3))
    for p in range(n):
        c = int(anchors[p]) if p < len(anchors) else int(rng.choice(anchors))
        k = int(rng.integers(views[0], views[1] + 1))
        turns = 2 if T > 1 and k >= 4 and rng.random() < 0.5 else 1
        t0 = min(c // P, T - turns)
        near = [c] + [t * P + (c % P + i) % P for i in range(P) for t in range(t0, t0 + turns)]
        vs = [v for v in dict.fromkeys(near) if v < V and ok[v]][:k]
        lists.append(np.sort(vs))
        r, th = 0.8 * np.sqrt(rng.random()), 2 * np.pi * rng.random()
        Pt[p] = [r * np.cos(th), 0.5 * (np.mean(vs) / P - T / 2) + rng.uniform(-0.3, 0.3), r * np.sin(th)]
    offsets = np.r_[0, np.cumsum([len(vs) for vs in lists])].astype(np.int64)
    view = np.concatenate(lists).astype(np.int32)
    track = np.repeat(np.arange(n), np.diff(offsets))
    _, r, _ = BO.reproject(Et[view], Kt[view], Pt[track], np.zeros((len(view), 2)))
    obs = r + noise * rng.standard_normal(r.shape)
    P0 = Pt * (1 + 0.01 * rng.standard_normal(Pt.shape))
    hold = np.zeros(n, bool)
    hold[list(held)] = True
    hold |= np.bincount(track, np.isin(view, held_views), n) > 0
    for p in np.flatnonzero(hold):
        E = ext32[lists[p][0]].astype(np.float64)
        P0[p] = E[:, :3].T @ (np.array([0.0, 0.0, -1.0]) - E[:, 3])
    return dict(points=P0, offsets=offsets, view=view, obs=obs, ext=ext32, intr=intr32), (Pt, Et, Kt), hold


def _depths(E, P, view, track):
    return (E[view, 2, :3] * P[track]).sum(1) + E[view, 2, 3]


@pytest.mark.parametrize("V,n,kw", [(2, 50, {}), (33, 400, {}), (40, 500, dict(unobserved=(1, 17, 39))),
                                    (256, 1500, dict(held=range(7), held_views=(5, 100, 200, 255))),
                                    (100, 600, dict(views=(2, 3)))])
def test_helix_scene_contract(V, n, kw):
    inp, (Pt, Et, _), hold = helix_scene(V, n, seed=V, **kw)
    lo, hi = kw.get("views", (3, 8))
    unobserved = kw.get("unobserved", ())
    view, track = inp["view"].astype(np.int64), np.repeat(np.arange(n), np.diff(inp["offsets"]))
    counts = np.diff(inp["offsets"])
    assert (counts >= min(lo, V - len(unobserved))).all() and (counts <= hi).all(), (counts.min(), counts.max())
    for t in range(n):                                              # one observation per view, in ascending view order
        assert (np.diff(view[inp["offsets"][t]:inp["offsets"][t + 1]]) > 0).all()
    per_view = np.bincount(view, minlength=V)
    assert (per_view[list(unobserved)] == 0).all()
    assert (np.delete(per_view, list(unobserved)) > 0).all()
    assert (_depths(Et, Pt, view, track) > 0).all()                 # the truth: every point in front of its cameras
    E0 = inp["ext"].astype(np.float64)
    front = _depths(E0, inp["points"], view, track) > 0             # the start, in the cameras handed in
    assert front[~hold[track]].all()
    assert not (np.bincount(track, ~front, n) > 0)[~hold].any() and (np.bincount(track, ~front, n) > 0)[hold].all()
    for v in kw.get("held_views", ()):
        assert hold[track[view == v]].all() and (view == v).any()
    assert np.array_equal(BO.Problem(inp["points"], inp["offsets"], inp["view"], inp["obs"], inp["ext"], inp["intr"]).incl,
                          ~hold)


# ------------------------------------------------------------------------------------------------------------------ cases
LOSSES = [("trivial", 1.0, True), ("trivial", 1.0, False), ("cauchy", 2.0, True), ("cauchy", 2.0, False)]

# name: (V, n, generator keywords, iterations, (loss, scale, refine_focal) settings).  The case of more tracks than the
# PCG grid's threads (200 k observations) runs 3 steps of about 350 PCG iterations each, at about 70 ms an iteration in the
# oracle, and the two settings that between them take each loss and each refine_focal once.
CASES = {
    # Two views with free focal lengths leave focal length against depth weakly constrained: at 4 units the oracle's PCG
    # iteration count over 12 steps moves by up to 4 under 1e-12 pixels of observation change.  The free-focal case puts the
    # cameras 1.5 units from the axis (depths 0.7 to 2.3, strong perspective) and stops after 4 steps, where it moves by 1.
    "V2": (2, 300, {}, 12, [LOSSES[1], LOSSES[3]]),
    "V2_free_focal": (2, 600, dict(distance=1.5), 4, [LOSSES[0], LOSSES[2]]),
    "V33": (33, 800, {}, 12, LOSSES),
    "V40_unobserved": (40, 1000, dict(unobserved=(1, 17, 39)), 15, LOSSES),
    "V128": (128, 1500, {}, 12, LOSSES),
    "V256": (256, 1500, {}, 12, LOSSES),
    "V256_held_views": (256, 2000, dict(held=range(7), held_views=(5, 100, 200, 255)), 12, LOSSES),
    "V256_36k_tracks": (256, 36000, {}, 3, [LOSSES[0], LOSSES[3]]),
}
BA_CASES = [(name, *s) for name, c in CASES.items() for s in c[4]]


@functools.lru_cache(maxsize=None)
def _scene(name):
    V, n, kw, _, _ = CASES[name]
    return helix_scene(V, n, seed=V + n, **kw)


@functools.lru_cache(maxsize=None)
def _oracle_run(name, loss, scale, refine_focal):
    inp, _, _ = _scene(name)
    return _oracle(inp, **_kw(name, loss, scale, refine_focal))


def _kw(name, loss, scale, refine_focal):
    return dict(iterations=CASES[name][3], refine_focal=refine_focal, loss=loss, loss_scale=scale)


def _idle_views(name):
    """Views with no refined observation: their cameras must come back as handed in."""
    inp, _, hold = _scene(name)
    track = np.repeat(np.arange(len(hold)), np.diff(inp["offsets"]))
    return np.setdiff1d(np.arange(CASES[name][0]), inp["view"][~hold[track]])


@pytest.mark.parametrize("name,loss,scale,refine_focal", BA_CASES)
def test_oracle_cases_converge(name, loss, scale, refine_focal):
    inp, _, hold = _scene(name)
    want = _oracle_run(name, loss, scale, refine_focal)
    print(f"{name} {loss} refine_focal={refine_focal}: status {want['status']}, {want['steps']} steps, "
          f"{want['pcg_iterations']} PCG iterations, cost {want['cost'][0]:.4g} -> {want['cost'][1]:.4g}")
    assert want["status"] in (0, 1) and want["steps"] >= 2
    assert want["cost"][1] < 0.5 * want["cost"][0] and np.all(np.diff(want["trace"]) <= 0)
    assert np.array_equal(want["points"][hold], inp["points"][hold]) and np.isinf(want["error"][hold]).all()
    idle = _idle_views(name)
    assert len(idle) == len(CASES[name][2].get("unobserved", ())) + len(CASES[name][2].get("held_views", ()))
    assert want["extrinsic"][idle].tobytes() == inp["ext"][idle].astype(np.float64).tobytes()
    assert want["intrinsic"][idle].tobytes() == inp["intr"][idle].astype(np.float64).tobytes()


def _nan_gradient_scene():
    """Two views, two tracks: track 0 observed exactly where the cameras handed in project its start (zero residual and
    gradient), track 1 with an observation at x = +inf, whose Cauchy weight is 0, so its gradient is 0 x inf = NaN and the cost
    +inf.  The untrained mini model's 48-view reconstruct below starts the same way: its focal lengths are +inf."""
    inp, _, _ = helix_scene(2, 2, seed=5, noise=0.0)
    track = np.repeat(np.arange(2), np.diff(inp["offsets"]))
    E, K = (inp[k].astype(np.float64)[inp["view"]] for k in ("ext", "intr"))
    inp["obs"] = BO.reproject(E, K, inp["points"][track], np.zeros((len(track), 2)))[1]
    inp["obs"][np.flatnonzero(track == 1)[0], 0] = np.inf
    return inp


def test_oracle_nan_gradient_is_not_small():
    got = _oracle(_nan_gradient_scene(), iterations=5, refine_focal=True, loss="cauchy", loss_scale=1.0)
    assert (got["status"], got["steps"], got["accepted"]) == (1, 5, 0)
    assert np.isinf(got["cost"]).all() and np.isinf(got["error"][1]) and got["error"][0] == 0.0


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_device_nan_gradient_is_not_small():
    """The gradient test took a NaN |g| for 0 (fmax drops NaNs) and stopped at once with status 0, "converged"."""
    inp = _nan_gradient_scene()
    kw = dict(iterations=5, refine_focal=True, loss="cauchy", loss_scale=1.0)
    _assert_matches(_device(inp, **kw), _oracle(inp, **kw), 5)


def _pcg_grid_bound(V):
    """The most CTAs ba_pcg_kernel's grid can have at V views: BA_VIEW_SMEM V doubles of dynamic shared memory, the 64-byte
    reduction buffer and the 1 KB the driver reserves per CTA, at most 2048 / 256 CTAs an SM; registers can only lower it."""
    props = torch.cuda.get_device_properties(0)
    smem = getattr(props, "shared_memory_per_multiprocessor", 233472)
    return min(2048 // 256, smem // (104 * 8 * V + 64 + 1024)) * props.multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("name,loss,scale,refine_focal", BA_CASES)
def test_device_matches_oracle_step_for_step(name, loss, scale, refine_focal):
    V, n, _, iterations, _ = CASES[name]
    inp, _, hold = _scene(name)
    kw = _kw(name, loss, scale, refine_focal)
    got = _device(inp, **kw)
    want = _oracle_run(name, loss, scale, refine_focal)
    pts, ext, intr = (t.cpu().numpy() for t in got[:3])
    steps, _, pcg, status = got[5].tolist()
    worst = max(max_rel_diff(a, b) for a, b in ((pts, want["points"]), (ext, want["extrinsic"]), (intr, want["intrinsic"])))
    ctas = _pcg_grid_bound(V)
    print(f"{name} {loss} refine_focal={refine_focal}: V={V} n={n} m={len(inp['view'])} steps={steps} status={status} "
          f"pcg={pcg} (oracle {want['pcg_iterations']}) worst rel diff {worst:.2e}; grid <= {ctas} CTAs: pass 2 "
          f"{V * 32} items / <= {ctas * 8} warps, pass 1 {n} tracks / <= {ctas * 256} threads")
    _assert_matches(got, want, iterations)
    idle = _idle_views(name)
    assert ext[idle].tobytes() == inp["ext"][idle].astype(np.float64).tobytes()
    assert intr[idle].tobytes() == inp["intr"][idle].astype(np.float64).tobytes()
    assert pts[hold].tobytes() == inp["points"][hold].tobytes()
    if V >= 128:
        assert V * 32 > ctas * 8                                   # pass 2: some warp takes more than one item
    if name == "V256_36k_tracks":
        assert n > ctas * 256                                      # pass 1 and the back-substitution loop per thread


@pytest.mark.gpu
def test_256_views_repeatable_and_poison_free():
    from test_poison_gpu import check_case
    inp, _, _ = _scene("V256_held_views")
    kw = _kw("V256_held_views", "cauchy", 2.0, True)
    a, b = _device(inp, **kw), _device(inp, **kw)
    for x, y in zip(a, b):
        assert torch.equal(x.view(-1).view(torch.uint8), y.view(-1).view(torch.uint8))
    check_case("bundle_adjust V=256", lambda P: _device(inp, **kw), finite=())


# ------------------------------------------------------------------------------------------------------------------ GPU: tracks, fused mesh
@pytest.mark.gpu
@pytest.mark.parametrize("S", [64, 96])
def test_tracks_of_long_surface_scenes(S):
    from test_tracks import _assert_equal, _oracle as tracks_oracle
    pairs = _ranking_pairs(S)
    got, pred, _ = _surface_tracks(S, pairs)
    want = tracks_oracle(pred, got, pairs, 2)
    print(f"tracks S={S}: {len(pairs)} ranking pairs, {len(want['points'])} tracks, {len(want['view'])} observations")
    assert len(want["points"]) > 1000 and len(np.unique(want["view"])) == S
    _assert_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,S,H,W,resolution,seed", [("two", 64, 60, 80, 200, 21), ("box", 96, 48, 64, 256, 22)])
def test_fused_mesh_of_long_scenes(kind, S, H, W, resolution, seed):
    from test_fused_mesh import _cuda, _device as fusion, assert_equal_to_oracle, oracle_of, synthetic_scene
    pred = _cuda(synthetic_scene(kind, S, H, W, seed=seed))
    res, tsdf, color = fusion(pred, resolution)
    want = oracle_of(pred, resolution)
    print(f"fused mesh {kind} S={S} {H}x{W} res={resolution}: grid {tuple(tsdf.shape)}, {len(want['indices'])} triangles")
    assert len(want["indices"]) > 0
    assert_equal_to_oracle(res, tsdf, color, want)


# ------------------------------------------------------------------------------------------------------------------ GPU: end to end
@pytest.mark.gpu
def test_reconstruct_48_views_tracks_bundle_adjust_fused_mesh():
    from omnivggt_official_b200 import ops
    from omnivggt_official_b200.geometry import compute_ranking
    from oracle.synth import make_inputs
    from test_fused_mesh import _device as fusion, assert_equal_to_oracle, oracle_of
    from test_model_gpu import model
    from test_tracks import _assert_equal, _oracle as tracks_oracle
    S = 48
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, S, 56, 56, seed=48).items()}
    rec = m.reconstruct(**inp, chunk=16, overlap=4)
    assert len(rec["chunks"]) >= 3
    e = torch.eye(4, device="cuda", dtype=torch.float64).repeat(S, 1, 1)
    e[:, :3] = rec["extrinsic"][0].double()
    ranking, _ = compute_ranking(e, k=6)
    pairs = [(i, int(r)) for i, row in enumerate(ranking.cpu().tolist()) for r in row if r != i]
    tr = m.tracks(rec, pairs, conf_percent=25.0)
    _assert_equal(tr, tracks_oracle(rec, tr, pairs, 2, pct=25.0))
    # The untrained model's focal lengths are +inf, which makes every residual and the cost +inf (that start is
    # test_device_nan_gradient_is_not_small's).  The adjustment takes the tracks and poses of the reconstruct with a finite
    # 56 x 56 pinhole instead, so it solves: a finite cost and accepted steps.
    assert torch.isinf(rec["intrinsic"][0, :, 0, 0]).all() and torch.isfinite(rec["extrinsic"]).all()
    K = torch.tensor([[56.0, 0.0, 28.0], [0.0, 56.0, 28.0], [0.0, 0.0, 1.0]], device="cuda").repeat(S, 1, 1)
    kw = dict(iterations=12, refine_focal=True, loss="cauchy", loss_scale=1.0)
    obs = tr["xy"].double() + 0.5
    got = ops.bundle_adjust(tr["points"], tr["offsets"], tr["view"], obs, tr["extrinsic"].contiguous(), K, trace=True, **kw)
    want = BO.bundle_adjust(*(t.cpu().numpy() for t in (tr["points"], tr["offsets"], tr["view"], obs, tr["extrinsic"], K)),
                            **kw)
    print(f"reconstruct S={S}: {len(rec['chunks'])} view sets, {len(pairs)} pairs, {len(tr['points'])} tracks, "
          f"{len(tr['view'])} observations, {int(want['problem'].incl.sum())} refined; bundle adjustment status "
          f"{want['status']}, {want['steps']} steps, {want['accepted']} accepted, {want['pcg_iterations']} PCG iterations, "
          f"cost {want['cost'][0]:.4g} -> {want['cost'][1]:.4g}")
    assert np.isfinite(want["cost"][0]) and want["accepted"] >= 1 and want["cost"][1] < want["cost"][0]
    _assert_matches(got, want, 12)
    # The reconstruct's own fused mesh is empty (its +inf focal lengths put every view's points on its optical axis, and
    # the untrained views carve each other): a structural check of the empty path.  With the pinhole the depth maps fuse.
    res, tsdf, color = fusion(rec, 100, 25.0)
    assert_equal_to_oracle(res, tsdf, color, oracle_of(rec, 100, 25.0))
    empty = len(res["indices"])
    pin = dict(rec, intrinsic=K[None])
    res, tsdf, color = fusion(pin, 100, 25.0)
    want = oracle_of(pin, 100, 25.0)
    print(f"fused mesh of the reconstruct: {empty} triangles; with the pinhole {len(want['indices'])}")
    assert empty == 0 and len(want["indices"]) > 0
    assert_equal_to_oracle(res, tsdf, color, want)
