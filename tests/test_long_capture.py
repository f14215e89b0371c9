"""Long captures: the view-set schedule, the Umeyama oracle against planted transforms and scipy, and the validation of
OmniVGGT.reconstruct (CPU); ovg_sim3_estimate / ovg_sim3_apply against the oracle and reconstruct end to end (GPU)."""
import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from oracle import sim3_oracle as SO
from oracle.make_golden_matches import surface_views


def _planted(rng, c=None, t_scale=1e3):
    R = Rotation.random(random_state=rng).as_matrix()
    c = float(10 ** rng.uniform(-3, 3)) if c is None else c
    t = rng.uniform(-t_scale, t_scale, 3)
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = c * R, t
    return M, R, c, t


def _map(M, p):
    return p @ M[:3, :3].T + M[:3, 3]


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max()


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("S", [1, 2, 7, 8, 9, 13, 20, 24, 25, 40, 48, 96, 97, 192])
@pytest.mark.parametrize("chunk,overlap", [(2, 1), (8, 1), (8, 3), (8, 4), (8, 7), (24, 8)])
def test_schedule(S, chunk, overlap):
    from omnivggt_official_b200.model import chunk_schedule
    ch = chunk_schedule(S, chunk, overlap)
    assert ch == SO.schedule(S, chunk, overlap)
    if S <= chunk:
        assert ch == [(0, S)]
        return
    assert all(b - a == chunk for a, b in ch)                                       # one graph signature
    assert ch[0][0] == 0 and ch[-1][1] == S
    seen = set()
    for k, (a, b) in enumerate(ch):
        if k:
            assert a > ch[k - 1][0] and b > ch[k - 1][1]
            assert ch[k - 1][1] - a >= overlap                                        # shares >= overlap views
        seen |= set(range(a, b))
    assert seen == set(range(S))
    assert [b - a for a, b in SO.new_views(ch)] and sum(b - a for a, b in SO.new_views(ch)) == S


def test_schedule_one_past_chunk():
    from omnivggt_official_b200.model import chunk_schedule
    assert chunk_schedule(9, 8, 3) == [(0, 8), (1, 9)]
    assert chunk_schedule(25, 24, 8) == [(0, 24), (1, 25)]
    assert chunk_schedule(40, 24, 8) == [(0, 24), (16, 40)]
    assert chunk_schedule(20, 8, 4) == [(0, 8), (4, 12), (8, 16), (12, 20)]


def test_aux_index_reindexing():
    from omnivggt_official_b200.model import chunk_index
    assert chunk_index([0, 3, 7, 8, 12], 5, 13) == [2, 3, 7] == SO.reindex([0, 3, 7, 8, 12], 5, 13)
    assert chunk_index(None, 0, 8) == [] and chunk_index([], 0, 8) == []
    assert chunk_index([4, 1], 0, 8) == [4, 1]                                       # order kept


@pytest.fixture()
def cpu_model(monkeypatch):
    """A small model on the CPU with the library replaced by a trap: validation must fail before any library call."""
    from omnivggt_official_b200 import _lib
    from omnivggt_official_b200.model import OmniVGGT

    def trap(*a, **k):
        raise AssertionError("library called before validation finished")
    monkeypatch.setattr(_lib, "lib", trap)
    m = OmniVGGT(img_size=56, embed_dim=128, depth=2, patch_embed="conv", dpt_features=128,
                 dpt_out_channels=(64, 128, 128, 128), dpt_layers=(0, 1, 0, 1), camera_heads=2, camera_trunk_depth=1)
    return m.eval()


@pytest.mark.parametrize("kw,exc", [
    (dict(images=torch.zeros(2, 10, 3, 56, 56)), ValueError),
    (dict(chunk=1, overlap=1), ValueError),
    (dict(chunk=8, overlap=0), ValueError),
    (dict(chunk=8, overlap=8), ValueError),
    (dict(chunk=8, overlap=9), ValueError),
    (dict(chunk=8.0), ValueError),
    (dict(conf_percent=-1.0), ValueError),
    (dict(conf_percent=100.5), ValueError),
    (dict(source="points"), ValueError),
    (dict(camera_gt_index=[10]), IndexError),
])
def test_reconstruct_validation(cpu_model, kw, exc):
    kw = dict(kw)
    images = kw.pop("images", torch.zeros(1, 10, 3, 56, 56))
    with pytest.raises(exc):
        cpu_model.reconstruct(images, **kw)


def test_reconstruct_validation_heads_and_cp(cpu_model):
    images = torch.zeros(10, 3, 56, 56)
    cpu_model.point_head = None
    with pytest.raises(ValueError):
        cpu_model.reconstruct(images, source="pointmap")
    cpu_model.camera_head = None
    with pytest.raises(ValueError):
        cpu_model.reconstruct(images)
    cpu_model._cp = object()
    with pytest.raises(RuntimeError):
        cpu_model.reconstruct(images)


@pytest.mark.parametrize("seed", range(8))
def test_oracle_recovers_planted_sim3(seed):
    rng = np.random.default_rng(seed)
    M, R, c, t = _planted(rng, c=[1e-3, 1e3, None][seed % 3])
    src = rng.standard_normal((500, 3)) * rng.uniform(0.1, 10, 3)
    sim3, st = SO.umeyama(src, _map(M, src))
    assert st[1] == 0 and st[0] == 500
    assert np.abs(sim3[:3, :3] / c - R).max() < 1e-12
    assert np.abs(sim3[:3, 3] - t).max() < 1e-12 * (np.abs(t).max() + c * np.abs(src).max())
    assert abs(st[3] / c - 1) < 1e-12 and np.linalg.det(sim3[:3, :3]) > 0


@pytest.mark.parametrize("case", ["planar", "three", "near_collinear", "mirror"])
def test_oracle_special_configurations(case):
    rng = np.random.default_rng(7)
    M, R, c, t = _planted(rng, c=2.5)
    if case == "planar":                # rank-2 covariance: det V is arbitrary, S must give a rotation
        src = np.c_[rng.standard_normal((200, 2)), np.zeros(200)]
    elif case == "three":
        src = rng.standard_normal((3, 3))
    elif case == "near_collinear":
        lam = rng.standard_normal(300)
        src = np.c_[lam, 2 * lam, -lam] + 1e-4 * rng.standard_normal((300, 3))
    else:                               # the target is a mirror image: the best proper rotation, never a reflection
        src = rng.standard_normal((400, 3))
        dst = src * [1, 1, -1]
        sim3, st = SO.umeyama(src, dst)
        assert st[1] == 0 and np.linalg.det(sim3[:3, :3]) > 0
        return
    sim3, st = SO.umeyama(src, _map(M, src))
    tol = 1e-8 if case == "near_collinear" else 1e-12
    assert st[1] == 0 and np.abs(sim3[:3, :3] / c - R).max() < tol and abs(st[3] / c - 1) < tol
    assert np.abs(sim3[:3, 3] - t).max() < tol * np.abs(t).max()


def test_oracle_degenerate_status():
    rng = np.random.default_rng(3)
    p = rng.standard_normal((50, 3))
    assert SO.umeyama(p[:2], p[:2])[1][1] == SO.STATUS_FEW
    assert SO.umeyama(p, p, keep=np.arange(50) < 2)[1][1] == SO.STATUS_FEW
    assert SO.umeyama(np.ones((50, 3)), p)[1][1] == SO.STATUS_SIGMA
    lam = np.arange(50.0)
    assert SO.umeyama(np.c_[lam, 2 * lam, 3 * lam], p)[1][1] == SO.STATUS_RANK
    bad = p.copy()
    bad[:48, 0] = np.nan
    sim3, st = SO.umeyama(bad, p)
    assert st[1] == SO.STATUS_FEW and st[0] == 2 and np.array_equal(sim3, np.eye(4)) and st[3] == 1


@pytest.mark.parametrize("seed", range(4))
def test_oracle_rotation_matches_align_vectors(seed):
    rng = np.random.default_rng(100 + seed)
    M, R, c, t = _planted(rng, c=0.7)
    src = rng.standard_normal((1000, 3))
    dst = _map(M, src) + 0.05 * rng.standard_normal((1000, 3))
    sim3, st = SO.umeyama(src, dst)
    rot, _ = Rotation.align_vectors(dst - dst.mean(0), src - src.mean(0))
    assert np.abs(sim3[:3, :3] / st[3] - rot.as_matrix()).max() < 1e-10
    assert np.abs(sim3[:3, :3] / st[3] - R).max() < 0.05


def test_extrinsic_update_identity_fp64():
    """unproject(c d, K, E') = c R unproject(d, K, E) + t in fp64, for the update of ovg_sim3_apply."""
    rng = np.random.default_rng(5)
    sv = surface_views(S=1, H=12, W=16, seed=2)
    d = sv[0, ..., 2][None].astype(np.float64)
    K = np.array([[[14.0, 0, 8], [0, 13.0, 6], [0, 0, 1]]])
    E = np.c_[Rotation.random(random_state=rng).as_matrix(), rng.standard_normal(3)][None]
    for c in (1e-3, 0.8, 37.0):
        M, _, _, _ = _planted(rng, c=c, t_scale=50)
        new = SO.apply(M, depth=d, ext=E, dtype=np.float64)
        lhs = SO.unproject(new["depth"], K, new["ext"])
        rhs = SO.apply(M, points=SO.unproject(d, K, E), dtype=np.float64)["points"]
        assert np.abs(lhs - rhs).max() < 1e-12 * np.abs(rhs).max()


# ------------------------------------------------------------------------------------------------------------------ GPU
def _cases():
    """name -> (src, dst, keep) fp32 / uint8 numpy: surface point maps under planted transforms."""
    rng = np.random.default_rng(21)
    out = {}
    sv = surface_views(S=2, H=48, W=64, seed=3).reshape(-1, 3)
    for i, c in enumerate((1e-3, 1.0, 1e3)):
        M, _, _, _ = _planted(rng, c=c)
        out[f"surface_c{c:g}"] = (sv, _map(M, sv.astype(np.float64)).astype(np.float32), None)
    M, _, _, _ = _planted(rng, c=3.0, t_scale=10)
    noisy = (_map(M, sv.astype(np.float64)) + 0.01 * rng.standard_normal(sv.shape)).astype(np.float32)
    out["noise"] = (sv, noisy, None)
    outl = noisy.copy()
    bad = rng.random(len(sv)) < 0.05
    outl[bad] += rng.uniform(-50, 50, (bad.sum(), 3)).astype(np.float32)
    out["outliers_masked"] = (sv, outl, (~bad).astype(np.uint8))
    out["outliers_unmasked"] = (sv, outl, None)
    nonf = noisy.copy()
    nonf[::97, 1] = np.nan
    nonf[5::101, 2] = np.inf
    src = sv.copy()
    src[7::89, 0] = -np.inf
    out["nan_inf"] = (src, nonf, None)
    for n in (3, 4, 255, 256, 257, 65535, 65536, 65537, 200_003, 4_194_304):
        p = (rng.standard_normal((n, 3)) * [3, 1, 0.5]).astype(np.float32)
        M, _, _, _ = _planted(rng)
        out[f"n{n}"] = (p, (_map(M, p.astype(np.float64)) + 1e-3 * rng.standard_normal((n, 3))).astype(np.float32),
                        (rng.random(n) < 0.9).astype(np.uint8) if n > 1000 else None)
    return out


CASES = _cases()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_align_sim3_matches_oracle(name):
    from omnivggt_official_b200 import geometry, ops
    src, dst, keep = CASES[name]
    ref, rst = SO.umeyama(src, dst, keep)
    got = geometry.align_sim3(src, dst, keep)
    assert got.dtype == torch.float64 and got.is_cuda and got.shape == (4, 4)
    g = got.cpu().numpy()
    assert _rel(g, ref) < 1e-9, (name, _rel(g, ref))
    s, d = (torch.from_numpy(x).cuda() for x in (src, dst))
    k = None if keep is None else torch.from_numpy(keep).cuda()
    m1, st1 = ops.sim3_estimate(s, d, k)
    m2, st2 = ops.sim3_estimate(s, d, k)
    assert torch.equal(m1, got) and torch.equal(m1, m2) and torch.equal(st1, st2)          # bit-identical
    st = st1.cpu().numpy()
    assert st[0] == rst[0] and st[1] == 0 and abs(st[3] / rst[3] - 1) < 1e-9
    assert abs(st[2] - rst[2]) <= 1e-9 * max(rst[2], 1e-30) + 1e-12 * np.abs(dst[np.isfinite(dst)]).max()


@pytest.mark.gpu
def test_align_sim3_degenerate_status():
    from omnivggt_official_b200 import geometry, ops
    rng = np.random.default_rng(9)
    p = rng.standard_normal((5000, 3)).astype(np.float32)
    lam = np.arange(5000, dtype=np.float32)[:, None]
    cases = {
        SO.STATUS_FEW: [(p[:2], p[:2], None), (p, p, (np.arange(5000) < 2).astype(np.uint8)),
                        (np.full_like(p, np.nan), p, None), (p[:0], p[:0], None)],
        SO.STATUS_SIGMA: [(np.full_like(p, 1.5), p, None)],
        SO.STATUS_RANK: [(lam * [1, 2, 3], p, None), (p, np.full_like(p, -2.0), None)],
    }
    for status, items in cases.items():
        for src, dst, keep in items:
            src, dst = np.ascontiguousarray(src, np.float32), np.ascontiguousarray(dst, np.float32)
            assert SO.umeyama(src, dst, keep)[1][1] == status
            k = None if keep is None else torch.from_numpy(keep).cuda()
            m, st = ops.sim3_estimate(torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda(), k)
            st = st.cpu().numpy()
            assert st[1] == status and np.array_equal(m.cpu().numpy(), np.eye(4)) and st[3] == 1.0, (status, st)
            with pytest.raises(ValueError):
                geometry.align_sim3(src, dst, keep)


@pytest.mark.gpu
def test_sim3_apply_is_fp64_rounded_once():
    from omnivggt_official_b200 import ops
    rng = np.random.default_rng(4)
    V, H, W = 3, 20, 28
    pts = (rng.standard_normal((V, H, W, 3)) * 5).astype(np.float32)
    pts2 = (rng.standard_normal((V, H, W, 3)) * 0.01).astype(np.float32)
    dep = rng.uniform(0.1, 50, (V, H, W, 1)).astype(np.float32)
    ext = np.c_[Rotation.random(V, random_state=rng).as_matrix(), rng.standard_normal((V, 3, 1))].astype(np.float32)
    for c in (1e-3, 0.77, 412.0):
        M, _, _, _ = _planted(rng, c=c)
        dev = [torch.from_numpy(x).cuda() for x in (pts, pts2, dep, ext)]
        outs = [torch.full_like(x, np.nan) for x in dev]
        ops.sim3_apply(torch.from_numpy(M).cuda(), V, H * W, points=[(dev[0], outs[0]), (dev[1], outs[1])],
                       depth=(dev[2], outs[2]), ext=(dev[3], outs[3]))
        ref = SO.apply(M, points=pts, depth=dep, ext=ext)
        assert np.array_equal(outs[0].cpu().numpy(), ref["points"])
        assert np.array_equal(outs[1].cpu().numpy(), SO.apply(M, points=pts2)["points"])
        assert np.array_equal(outs[2].cpu().numpy(), ref["depth"])
        assert np.array_equal(outs[3].cpu().numpy(), ref["ext"])


def _device_threshold(pct):
    from omnivggt_official_b200 import ops
    return lambda conf: ops.conf_percentile_mask(torch.from_numpy(np.ascontiguousarray(conf)).cuda(), pct, 1e-5)[1].item()


def _raw_chunk(m, inp, a, b, didx, cidx):
    """model(...) on views a..b-1 with the re-indexed aux lists, decoded and unprojected, as numpy."""
    from omnivggt_official_b200 import ops
    from omnivggt_official_b200.model import chunk_index
    H, W = inp["images"].shape[-2:]
    raw = m(**{k: v[:, a:b] for k, v in inp.items()}, depth_gt_index=chunk_index(didx, a, b),
            camera_gt_index=chunk_index(cidx, a, b))
    ext, intr, c2w = ops.pose_decode(raw["pose_enc"][0].float().contiguous(), H, W)
    wpd = ops.unproject_depth(raw["depth"][0].float().reshape(b - a, H, W), intr, c2w, H, W)
    out = {"extrinsic": ext, "intrinsic": intr, "depth": raw["depth"][0], "depth_conf": raw["depth_conf"][0],
           "world_points_from_depth": wpd, "world_points": raw["world_points"][0],
           "world_points_conf": raw["world_points_conf"][0]}
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("S,overlap,aux", [(5, 3, False), (5, 1, True), (13, 1, False), (13, 3, True), (13, 4, False),
                                           (20, 1, True), (20, 3, False), (20, 4, True), (20, 4, False)])
def test_reconstruct_mini(S, overlap, aux, tmp_path):
    from test_model_gpu import model
    from omnivggt_official_b200.glb import write_glb
    from omnivggt_official_b200.model import OmniVGGT
    from oracle.synth import make_inputs
    m = model("mini_conv")
    chunk = 8
    inp = {k: v.cuda() for k, v in make_inputs(1, S, 56, 56, seed=50 + S).items()}
    didx = [i for i in (1, 6, 7, 9, 15) if i < S] if aux else None          # lists that span view-set boundaries
    cidx = [i for i in (0, 7, 8, 12, 19) if i < S] if aux else None
    out = m.reconstruct(**inp, depth_gt_index=didx, camera_gt_index=cidx, chunk=chunk, overlap=overlap)
    chunks = SO.schedule(S, chunk, overlap)
    assert out["chunks"] == chunks and out["sim3"].shape == (len(chunks), 4, 4) and out["sim3"].dtype == torch.float64
    assert "pose_enc" not in out and out["images"] is inp["images"]
    raws = {c: _raw_chunk(m, inp, *c, didx, cidx) for c in chunks}
    got = {k: out[k][0].cpu().numpy() for k in SO.POINT_KEYS + SO.COPY_KEYS + ("depth", "extrinsic")}
    sims = out["sim3"].cpu().numpy()
    ref = SO.merge(lambda a, b: raws[(a, b)], S, chunk, overlap, threshold=_device_threshold(50.0))
    for k, ((a, b), (n0, n1)) in enumerate(zip(chunks, SO.new_views(chunks))):
        r, new = raws[(a, b)], slice(n0 - a, b - a)
        if k == 0:
            assert np.array_equal(sims[0], np.eye(4))
            for key in got:
                assert np.array_equal(got[key][a:b], r[key]), key                   # chunk 0 = the plain forward
            continue
        assert _rel(sims[k], ref["sim3"][k]) < 1e-9, (k, _rel(sims[k], ref["sim3"][k]))
        assert out["align_pairs"][k].item() == ref["align_pairs"][k] > 0
        want = SO.apply(sims[k], depth=r["depth"][new], ext=r["extrinsic"][new])
        assert np.array_equal(got["depth"][n0:n1], want["depth"])
        assert np.array_equal(got["extrinsic"][n0:n1], want["ext"])
        for key in SO.POINT_KEYS:
            assert np.array_equal(got[key][n0:n1], SO.apply(sims[k], points=r[key][new])["points"]), key
        for key in SO.COPY_KEYS:
            assert np.array_equal(got[key][n0:n1], r[key][new]), key
    assert out["align_pairs"][0] == 0 and out["align_rmse"][0] == 0
    # the merged depth unprojected through the merged cameras lands on the merged points
    re = SO.unproject(got["depth"][..., 0], got["intrinsic"], got["extrinsic"])
    p = got["world_points_from_depth"]
    assert np.abs(re - p).max() < 2e-4 * np.abs(p).max(), np.abs(re - p).max()
    cloud = OmniVGGT.point_cloud(out, conf_percent=20.0)
    assert cloud["points"].shape[0] > 0 and set(cloud["frame"].unique().tolist()) <= set(range(S))
    mesh = OmniVGGT.mesh(out, layout="glb")
    assert mesh["indices"].shape[0] > 0
    assert OmniVGGT.sky_mask(out).shape == (S, 56, 56)
    assert len(OmniVGGT.matches(out, [(0, S - 1)])) == 1
    write_glb(str(tmp_path / "scene.glb"), cloud)
    assert (tmp_path / "scene.glb").stat().st_size > 0


@pytest.mark.gpu
def test_reconstruct_pointmap_source_and_single_chunk():
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 13, 56, 56, seed=77).items()}
    out = m.reconstruct(**inp, chunk=8, overlap=3, source="pointmap", conf_percent=30.0)
    raws = {c: _raw_chunk(m, inp, *c, None, None) for c in out["chunks"]}
    ref = SO.merge(lambda a, b: raws[(a, b)], 13, 8, 3, source="pointmap", conf_percent=30.0,
                   threshold=_device_threshold(30.0))
    for k in range(1, len(out["chunks"])):
        assert _rel(out["sim3"][k].cpu().numpy(), ref["sim3"][k]) < 1e-9
    one = m.reconstruct(**{k: v[:, :6] for k, v in inp.items()}, chunk=8, overlap=3)      # S <= chunk: the plain forward
    r = _raw_chunk(m, {k: v[:, :6] for k, v in inp.items()}, 0, 6, None, None)
    assert one["chunks"] == [(0, 6)] and torch.equal(one["sim3"][0].cpu(), torch.eye(4, dtype=torch.float64))
    for key, v in r.items():
        assert np.array_equal(one[key][0].cpu().numpy(), v), key


@pytest.mark.gpu
def test_reconstruct_full_size_graph_replay_bit_identical():
    """The full architecture at 518 x 518, S = 40 as two view sets of 24 sharing 8: eager forwards and CUDA-graph replays
    give the same merged scene bit for bit."""
    from omnivggt_official_b200 import OmniVGGT
    from oracle.synth import make_inputs
    with torch.device("cuda"):
        m = OmniVGGT(init_seed=None)
    m.randomize_(0).eval()
    inp = {k: v.cuda() for k, v in make_inputs(1, 40, 518, 518, seed=6).items()}
    m.use_cuda_graph = False
    eager = m.reconstruct(inp["images"], chunk=24, overlap=8)
    m.use_cuda_graph = True
    m.reconstruct(inp["images"], chunk=24, overlap=8)                    # calls 1 and 2 of the signature run eagerly
    graphed = m.reconstruct(inp["images"], chunk=24, overlap=8)          # call 3 captures, call 4 replays
    assert eager["chunks"] == [(0, 24), (16, 40)]
    for k in ("extrinsic", "intrinsic", "depth", "depth_conf", "world_points_from_depth", "world_points",
              "world_points_conf", "sim3", "align_pairs", "align_rmse"):
        assert torch.equal(eager[k], graphed[k]), k
    for k in ("depth", "world_points_from_depth", "sim3"):          # random weights: focal lengths may overflow to inf
        assert torch.isfinite(eager[k]).all(), k
    assert eager["align_pairs"][1] > 0
    del m
    torch.cuda.empty_cache()
