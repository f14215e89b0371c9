"""The full-size fixtures and their checker (oracle/full_golden.py), without a GPU.

The checker must have the power the GPU tests rely on: a golden plus noise at the error level measured on the H100 passes,
and each seeded mistake of the kind a kernel bug makes (one view off by a few percent, a wrong border line, a DPT chunk
offset, one bad camera) fails and names the view, line or output it was seeded in.  The fixtures must sample exactly the
configurations bench.py measures, including the image borders and every position inside a 14-pixel patch."""
import os

import pytest
import torch

from bench import CONFIGS
from oracle.full_golden import BARS, DENSE, GOLDEN, PATCH, check, compare, index, lines, load, sample

INDEX = index()
CASES = sorted(INDEX)
BENCH_CASES = {"full_cfg1": "cfg1", "full_cfg2": "cfg2", "full_cfg3": "cfg3", "full_cfg5": "cfg5"}
# Worst rel-L2 of an output over one view or border line, over all full-size cases on the H100 with the fp16 heads
# (DESIGN.md §2).
MEASURED_REL = 7.7e-3


def noisy(ref, case):
    """The fixture plus seeded noise of rel-L2 MEASURED_REL on every output: what a correct kernel path returns.  Dense maps
    get it per value (as rounding does), pose encodings scaled by their RMS, so small entries are not held to a relative bar."""
    g = torch.Generator().manual_seed(CASES.index(case))
    got = {}
    for k, v in ref.items():
        u = (torch.rand(v.shape, generator=g, dtype=torch.float64) * 2 - 1) * 3 ** 0.5      # unit variance
        scale = v if k in DENSE else v.double().pow(2).mean().sqrt()
        got[k] = (v + MEASURED_REL * scale * u).float()
    return got


@pytest.fixture(scope="module", params=CASES)
def case(request):
    return request.param, INDEX[request.param], load(request.param)


def test_noise_at_measured_level_passes(case):
    name, meta, ref = case
    check(compare(noisy(ref, name), ref, meta))
    check(compare(ref, ref, meta))


def test_one_view_three_percent_off_fails_naming_the_view(case):
    name, meta, ref = case
    S, v = meta["S"], meta["S"] - 2
    got, off = noisy(ref, name), dict(ref)
    for k in DENSE:
        got[k][:, v] *= 1.03
        off[k] = ref[k].clone()
        off[k][:, v] *= 1.03
    if S >= 24:     # what one number per output misses
        agg = compare(off, ref, meta)["aggregate"]
        assert all(agg[k] < BARS["aggregate"] for k in DENSE), agg
    with pytest.raises(AssertionError) as e:
        check(compare(got, ref, meta))
    for k in DENSE:
        assert f"{k}: view {v} rel-L2" in str(e.value) and f"(views over the bar: [{v}])" in str(e.value)


def test_row0_replaced_by_row1_fails_naming_the_border_line(case):
    name, meta, ref = case
    got = noisy(ref, name)
    assert meta["rows"][:2] == [0, 1]
    for k in DENSE:
        got[k][:, :, 0] = got[k][:, :, 1]
    with pytest.raises(AssertionError) as e:
        check(compare(got, ref, meta))
    for k in DENSE:       # row 0 is the worst line; a column line holds one changed sample per view and may be over too
        assert f"{k}: border row 0 rel-L2" in str(e.value)
    assert "row 1" not in str(e.value) and "row 51" not in str(e.value)


def test_pose_enc_of_one_view_off_by_0p1_fails_naming_the_view(case):
    name, meta, ref = case
    v = meta["S"] // 2
    got = noisy(ref, name)
    got["pose_enc"][:, v, 0] += 0.1
    with pytest.raises(AssertionError, match=rf"pose_enc: view {v} max-abs") as e:
        check(compare(got, ref, meta))
    assert f"views over the bar: [{v}]" in str(e.value)


def test_dpt_chunk_offset_fails_naming_the_views():
    """Views 8..15 of full_cfg5 rotated by one (the second 8-frame DPT chunk reading its frames one view late)."""
    meta, ref = INDEX["full_cfg5"], load("full_cfg5")
    got = noisy(ref, "full_cfg5")
    for k in DENSE:
        got[k][:, 8:16] = torch.roll(got[k][:, 8:16], 1, dims=1)
    with pytest.raises(AssertionError) as e:
        check(compare(got, ref, meta))
    for k in DENSE:
        assert f"{k}: view " in str(e.value) and "(views over the bar: [8, 9, 10, 11, 12, 13, 14, 15])" in str(e.value)


# ------------------------------------------------------------------------------------------------ fixture integrity
@pytest.mark.parametrize("name,cfg", sorted(BENCH_CASES.items()))
def test_index_lists_are_the_benchmarks(name, cfg):
    meta, c = INDEX[name], CONFIGS[cfg]
    assert (meta["S"], meta["depth_gt_index"], meta["camera_gt_index"]) == (c["S"], c["depth_idx"], c["cam_idx"])
    assert (meta["H"], meta["W"]) == (518, 518)


def test_fixture_layout(case):
    name, meta, ref = case
    H, W, S = meta["H"], meta["W"], meta["S"]
    rows, cols = meta["rows"], meta["cols"]
    assert rows == lines(H, meta["stride"], meta["offset"]) and cols == lines(W, meta["stride"], meta["offset"])
    for ln, n in ((rows, H), (cols, W)):
        assert {0, 1, n - 2, n - 1} <= set(ln) and ln == sorted(set(ln)) and 0 <= ln[0] and ln[-1] < n
    assert ref["pose_enc"].shape == (1, S, 9) and all(ref[f"pose_enc_list.{i}"].shape == (1, S, 9) for i in range(4))
    for k, c in zip(DENSE, (1, None, 3, None)):
        assert ref[k].shape == (1, S, len(rows), len(cols)) + ((c,) if c else ()), k
        assert torch.isfinite(ref[k]).all(), k
    assert os.path.getsize(os.path.join(GOLDEN, f"{name}.safetensors")) < 1e6
    assert meta["cpu_forward_s"] > 0


@pytest.mark.parametrize("name", ["full_cfg2", "full_cfg3", "full_cfg5", "full_land_s10", "full_wide_s5", "full_tall_s3"])
def test_new_cases_cover_every_position_in_a_patch(name):
    meta = INDEX[name]
    for ln, n in ((meta["rows"], meta["H"]), (meta["cols"], meta["W"])):
        assert {x % PATCH for x in ln if 1 < x < n - 2} == set(range(PATCH))


@pytest.mark.parametrize("name,H,W", [("full_land_s10", 392, 518), ("full_wide_s5", 294, 518), ("full_tall_s3", 882, 518)])
def test_non_square_cases_are_the_loader_shapes(name, H, W):
    """4:3 and 16:9 photos and the tallest input the engine accepts, as the loaders produce them (width 518, height scaled)."""
    assert (INDEX[name]["H"], INDEX[name]["W"]) == (H, W)


def test_sample_takes_the_listed_rows_and_columns():
    B, S, H, W = 2, 3, 20, 18
    rows, cols = lines(H, 7, 3), lines(W, 5, 4)
    base = torch.arange(B * S * H * W, dtype=torch.float32).reshape(B, S, H, W)
    out = {"pose_enc": torch.randn(B, S, 9), "pose_enc_list": [torch.randn(B, S, 9) for _ in range(4)],
           "depth": base[..., None], "depth_conf": base + 1, "world_points": torch.stack([base, -base, 2 * base], -1),
           "world_points_conf": base + 2}
    got = sample(out, rows, cols)
    for i, y in enumerate(rows):
        for j, x in enumerate(cols):
            assert torch.equal(got["depth"][:, :, i, j, 0], base[:, :, y, x])
            assert torch.equal(got["world_points"][:, :, i, j], out["world_points"][:, :, y, x])
    assert torch.equal(got["pose_enc_list.3"], out["pose_enc_list"][3])
