"""Image ranking by camera distance: the numpy oracle against the unmodified reference's compute_ranking (CPU), the
validation and call pattern of the drop-in on a recorded library (CPU), and the libovg kernels against the goldens and the
oracle on both regimes (GPU)."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import ranking_oracle as RO
from oracle.make_golden_ranking import make_cases, poses, trajectory
from ovg_support import install, sha256

CASES = make_cases()
CTA = 8192           # OVG_RANK_CTA_VIEWS: one CTA per row with the keys in shared memory up to here, the grid above


def _meta():
    with open(os.path.join(GOLDEN, "ranking.json")) as f:
        return json.load(f)


def _gold(name):
    with np.load(os.path.join(GOLDEN, "ranking.npz")) as z:
        return z[f"{name}.dists"], z[f"{name}.ranking"].astype(np.int64)


def _truth(k, rows=None):
    return RO.truth(k["E"], k["lambda_t"], k["normalize"], k["batched"], chunked=k["chunk"] is not None, rows=rows)


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_inputs_are_reproduced(name):
    m = _meta()[name]
    E = CASES[name]["E"]
    assert sha256(E) == m["E_sha256"]
    assert list(E.shape) == m["E_shape"] and str(E.dtype) == m["E_dtype"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_lies_within_the_oracle_bound(name):
    k = CASES[name]
    ref_d, ref_rank = _gold(name)
    tr = _truth(k)
    assert ref_d.dtype == tr["out"] == np.dtype(_meta()[name]["dists_dtype"])
    b = RO.bound(tr)
    nan = np.isnan(tr["d"])
    assert np.array_equal(nan, np.isnan(ref_d))
    err = np.abs(ref_d.astype(np.float64) - tr["d"])
    assert (err[~nan] <= b[~nan]).all(), (err - b).max()
    oracle_rank = np.argsort(tr["d"].astype(tr["out"]), axis=1, kind="stable")
    assert RO.ranking_agrees(ref_d, ref_rank, b, oracle_rank).all()


def test_oracle_bound_is_tight_enough_to_check_rankings():
    """Random poses are far apart against the bound: almost every position of their rankings is checked."""
    k = CASES["f64"]
    ref_d, ref_rank = _gold("f64")
    assert RO.isolated(ref_d, ref_rank, RO.bound(_truth(k))).mean() > 0.95
    k = CASES["f32"]
    ref_d, ref_rank = _gold("f32")
    assert RO.isolated(ref_d, ref_rank, RO.bound(_truth(k))).mean() > 0.8


def test_kernel_scale_restatement_is_a_fixed_order_mean():
    t = np.random.default_rng(3).standard_normal((1000, 3))
    nrm = np.sqrt((t * t).sum(1))
    assert abs(RO.mean_norm(t) - nrm.mean()) <= 1e-14 * nrm.mean()


@pytest.mark.parametrize("name", ["f64", "f32_lambda2p5", "chunked_f64", "chunked_f32_lambda2p5"])
def test_numpy_restatement_matches_the_reference(name):
    k = CASES[name]
    ref_d, _ = _gold(name)
    _, d = RO.reference_numpy(k["E"], k["lambda_t"], k["normalize"], chunk=k["chunk"])
    assert d.dtype == ref_d.dtype and np.allclose(d, ref_d, rtol=0, atol=1e-5 if d.dtype == np.float32 else 1e-12)


@pytest.fixture()
def dry(monkeypatch):
    """The C library replaced by a recorder, on CPU tensors; host reads recorded."""
    from omnivggt_official_b200 import geometry
    fake = install(monkeypatch)
    monkeypatch.setattr(geometry, "_device_of", lambda *xs: torch.device("cpu"))
    return fake


@pytest.mark.parametrize("N,dtype,batched,out", [(50, np.float64, True, torch.float64), (50, np.float32, True, torch.float32),
                                                 (50, np.float32, False, torch.float64),
                                                 (6000, np.float64, True, torch.float64),
                                                 (6001, np.float64, True, torch.float32),
                                                 (6001, np.float64, False, torch.float64)])
def test_dry_run_is_one_call_without_host_read(dry, N, dtype, batched, out):
    from omnivggt_official_b200.geometry import compute_ranking
    E = np.zeros((N, 4, 4), dtype)
    for k in (None, 1, 7, N):
        for lam, normalize in ((1.0, True), (0.1, False)):
            dry.calls.clear()
            ranking, dists = compute_ranking(E, lambda_t=lam, normalize=normalize, batched=batched, k=k)
            assert dry.names() == ["ovg_ranking_workspace_bytes", "ovg_compute_ranking"]
            assert dry.calls[0][1] == (N, int(out == torch.float64))
            a = dry.calls[1][1]
            f32_compute = dtype == np.float32 or out == torch.float32
            assert a[1:6] == (int(dtype == np.float64), N, 16, 4, 1)
            assert a[6] == (float(np.float32(lam)) if f32_compute else lam)
            assert a[7:10] == (int(normalize), int(out == torch.float64), N if k is None else k)
            assert ranking.shape == (N, N if k is None else k) and ranking.dtype == torch.int64
            assert dists.shape == (N, N) and dists.dtype == out


def test_dry_run_passes_strides_of_a_view(dry):
    """A [S, 3, 4] slice of a batch of 4x4 extrinsics goes in with its strides, uncopied."""
    from omnivggt_official_b200.geometry import compute_ranking
    E = torch.zeros(2, 9, 4, 4)[0, :, :3]
    compute_ranking(E)
    a = dry.calls[1][1]
    assert a[0] == E.data_ptr() and a[1:6] == (0, 9, 16, 4, 1)


def test_n0_returns_empty_outputs(dry):
    from omnivggt_official_b200.geometry import compute_ranking
    for dtype, batched, out in ((np.float32, True, torch.float32), (np.float64, True, torch.float64),
                                (np.float32, False, torch.float64)):
        ranking, dists = compute_ranking(np.zeros((0, 4, 4), dtype), batched=batched)
        assert ranking.shape == (0, 0) and ranking.dtype == torch.int64
        assert dists.shape == (0, 0) and dists.dtype == out
    assert dry.calls == []


def test_errors_before_any_library_call(dry):
    from omnivggt_official_b200.geometry import compute_ranking
    E = np.zeros((5, 4, 4))
    for ext, k, what in ((np.zeros((5, 16)), None, "shape"), (np.zeros((5, 4, 4, 1)), None, "shape"),
                         (np.zeros((5, 2, 4)), None, "shape"), (np.zeros((5, 4, 3)), None, "shape"),
                         (np.zeros((5, 4, 4), np.float16), None, "dtype"), (np.zeros((5, 4, 4), np.int64), None, "dtype"),
                         (torch.zeros(5, 4, 4, dtype=torch.bfloat16), None, "dtype"), (E, 0, "k"), (E, 6, "k"),
                         (E, -1, "k"), (E, 2.0, "k"), (E, True, "k"), (np.zeros((0, 4, 4)), 1, "k")):
        with pytest.raises(ValueError, match=what):
            compute_ranking(ext, k=k)
    assert dry.calls == []


# ------------------------------------------------------------------------------------------------------------------ GPU
def _run(k, kk=None):
    """The drop-in, or for a chunked case the library at fp32 output (the chunked formula at small N)."""
    from omnivggt_official_b200 import ops
    from omnivggt_official_b200.geometry import compute_ranking
    E = torch.from_numpy(k["E"]).cuda()
    if k["chunk"] is None:
        return compute_ranking(E, k["lambda_t"], k["normalize"], k["batched"], k=kk)
    lam = RO.kernel_lambda(k["lambda_t"], np.float32)
    return ops.compute_ranking(E, lam, k["normalize"], torch.float32, E.shape[0] if kk is None else kk)


def _self_consistent(ranking, dists):
    return torch.equal(ranking, torch.argsort(dists, dim=1, stable=True))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_kernel_matches_golden(name):
    k = CASES[name]
    ref_d, ref_rank = _gold(name)
    ranking, dists = _run(k)
    assert dists.dtype == getattr(torch, str(ref_d.dtype)) and ranking.dtype == torch.int64
    assert _self_consistent(ranking, dists)
    tr = _truth(k)
    got = dists.cpu().numpy()
    assert RO.within_ulps(got, tr).all(), np.argwhere(~RO.within_ulps(got, tr))[:5]
    assert RO.ranking_agrees(ref_d, ref_rank, RO.bound(tr), ranking.cpu().numpy()).all()
    if len(ref_d) > 2:
        top, _ = _run(k, 3)
        assert torch.equal(top, ranking[:, :3])


def _large(N, seed):
    rng = np.random.default_rng(seed)
    E = poses(rng, N, np.float64)
    E[::5] = trajectory(len(E[::5]), np.float64)               # a dense video through random views
    E[7::97] = E[3]                                             # duplicated poses: ties
    return E


LARGE = {          # N, batched: the reference's dtype rule gives fp32 dists above 6000 views batched, fp64 unbatched
    "smem_at_threshold_f32": (CTA, True),
    "smem_at_threshold_f64": (CTA, False),
    "grid_above_threshold_f32": (CTA + 1, True),
    "grid_above_threshold_f64": (CTA + 1, False),
    "smem_6000_f64": (6000, True),
    "smem_6001_f32": (6001, True),
    "grid_20000_f32": (20000, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LARGE))
def test_large_n(name):
    from omnivggt_official_b200.geometry import compute_ranking
    N, batched = LARGE[name]
    E = _large(N, seed=N)
    ranking, dists = compute_ranking(torch.from_numpy(E).cuda(), batched=batched)
    assert dists.dtype == (torch.float64 if not batched or N <= 6000 else torch.float32)
    assert _self_consistent(ranking, dists)
    rows = np.sort(np.random.default_rng(1).choice(N, 64, replace=False))
    rows[:2] = (0, N - 1)
    tr = RO.truth(E, 1.0, True, batched, rows=rows)
    got = dists[torch.from_numpy(rows).cuda()].cpu().numpy()
    assert RO.within_ulps(got, tr).all(), np.argwhere(~RO.within_ulps(got, tr))[:5]
    top, dists64 = compute_ranking(torch.from_numpy(E).cuda(), batched=batched, k=64)
    assert torch.equal(top, ranking[:, :64])
    assert torch.equal(dists64, dists)
    again, dists2 = compute_ranking(torch.from_numpy(E).cuda(), batched=batched)
    assert torch.equal(again, ranking) and torch.equal(dists2, dists)


@pytest.mark.gpu
def test_extrinsic_views_and_non_finite_rows():
    """A strided [S, 3, 4] view as the model predicts it, negative distances, a duplicated pose, and a NaN pose: its row
    is all NaN in index order and it sorts last in every other row."""
    from omnivggt_official_b200.geometry import compute_ranking
    E = torch.from_numpy(poses(np.random.default_rng(4), 300, np.float32)).cuda()
    E[10] = E[11]
    E[20, 0, 0] = float("nan")
    pred = torch.zeros(1, 300, 4, 4, device="cuda")
    pred[0] = E
    view = pred[0, :, :3]
    assert not view.is_contiguous()
    ranking, dists = compute_ranking(view, lambda_t=-1.0, normalize=False)
    ref, dref = compute_ranking(E.contiguous())
    want = RO.truth(E.cpu().numpy(), -1.0, False)
    assert RO.within_ulps(dists.cpu().numpy(), want).all()
    assert _self_consistent(ranking, dists) and _self_consistent(ref, dref)
    assert torch.isnan(dists[20]).all() and torch.equal(ranking[20], torch.arange(300, device="cuda"))
    assert (ranking[:, -1] == 20).sum() == 299
