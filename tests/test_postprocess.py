"""Post-processing (SURVEY.md section 8f rank 3): the numpy oracle against outputs of the unmodified reference functions
(CPU), and the libovg kernels against the oracle and the same golden (GPU, through the C ABI)."""
import os

import numpy as np
import pytest
import torch
from safetensors.torch import load_file

from conftest import GOLDEN
from oracle import postprocess_oracle as PO
from oracle.make_golden_post import make_post_inputs

PCTS = (0.0, 37.5, 50.0, 99.9, 100.0)


def _gold():
    return load_file(os.path.join(GOLDEN, "postprocess.safetensors"))


def test_oracle_matches_reference_postprocessing():
    g = _gold()
    pose, depth, conf = make_post_inputs()
    H, W = depth.shape[2:4]
    ext, intr = PO.pose_encoding_to_extri_intri(pose.numpy(), H, W)
    assert np.allclose(ext, g["extrinsic"].numpy(), rtol=1e-5, atol=1e-6)
    assert np.allclose(intr, g["intrinsic"].numpy(), rtol=1e-5, atol=1e-4)
    world = PO.unproject_depth_map_to_point_map(depth[0, ..., 0].numpy(), ext[0], intr[0])
    ref = g["world_points_from_depth"].numpy()
    assert np.abs(world - ref).max() <= 1e-4 * np.abs(ref).max()
    for pct in PCTS:
        mask, thr = PO.conf_percentile_mask(conf.numpy(), pct)
        assert float(thr) == float(g[f"thr_{pct}"]) and np.array_equal(mask.reshape(-1), g[f"mask_{pct}"].numpy().astype(bool))


@pytest.mark.gpu
def test_pose_decode_and_unproject_kernels():
    from omnivggt_official_b200 import ops
    g = _gold()
    pose, depth, conf = make_post_inputs()
    H, W = depth.shape[2:4]
    ext, intr, c2w = ops.pose_decode(pose.cuda(), H, W)
    torch.cuda.synchronize()
    assert torch.allclose(ext.cpu(), g["extrinsic"], rtol=1e-5, atol=2e-6)
    assert torch.allclose(intr.cpu(), g["intrinsic"], rtol=2e-5, atol=1e-4)
    c2w_ref = PO.se3_inverse_3x4(g["extrinsic"].numpy())
    assert np.allclose(c2w.cpu().numpy(), c2w_ref, rtol=1e-5, atol=1e-5)
    S = depth.shape[1]
    world = ops.unproject_depth(depth[0, ..., 0].cuda(), intr.view(S, 3, 3), c2w.view(S, 3, 4), H, W)
    torch.cuda.synchronize()
    ref = g["world_points_from_depth"]
    err = (world.cpu() - ref).abs().max().item()
    assert err <= 2e-5 * ref.abs().max().item(), err          # fp32 vs the reference's numpy fp32/fp64 mix
    # odd width: scalar path
    d2 = depth[0, :, :, :69, 0].contiguous().cuda()
    w2 = ops.unproject_depth(d2, intr.view(S, 3, 3), c2w.view(S, 3, 4), H, 69)
    ref2 = PO.unproject_depth_map_to_point_map(d2.cpu().numpy(), ext[0].cpu().numpy(), intr[0].cpu().numpy())
    assert np.abs(w2.cpu().numpy() - ref2).max() <= 2e-5 * np.abs(ref2).max()


@pytest.mark.gpu
@pytest.mark.parametrize("pct", PCTS)
def test_conf_percentile_mask_kernel_is_exact(pct):
    """Exact order statistics and numpy's fp32 interpolation: the threshold and the mask equal the reference's."""
    from omnivggt_official_b200 import ops
    g = _gold()
    _, _, conf = make_post_inputs()
    mask, thr, cnt = ops.conf_percentile_mask(conf.cuda(), pct)
    torch.cuda.synchronize()
    t_ref = float(g[f"thr_{pct}"])
    assert thr.item() == t_ref, (thr.item(), t_ref)
    got = mask.cpu().reshape(-1).bool()
    assert torch.equal(got, g[f"mask_{pct}"].bool())
    assert int(cnt.item()) == int(got.sum())


@pytest.mark.gpu
def test_conf_percentile_large_with_negatives_and_ties():
    """2.1 M values (8 views @ 518^2) incl. negatives, zeros and heavy ties; odd length exercises the scalar tail."""
    from omnivggt_official_b200 import ops
    g = torch.Generator().manual_seed(5)
    v = torch.randn(8 * 518 * 518 + 3, generator=g)
    v[::7] = 0.0
    v[1::11] = v[1].item()
    vc = v.cuda()
    for pct in (12.5, 50.0, 90.0):
        mask, thr, cnt = ops.conf_percentile_mask(vc, pct, floor=-1e30)
        t_ref = np.percentile(v.numpy(), pct)
        assert thr.item() == float(t_ref), (thr.item(), t_ref)
        ref_mask = torch.from_numpy(v.numpy() >= t_ref)
        assert torch.equal(mask.cpu().bool(), ref_mask) and int(cnt.item()) == int(ref_mask.sum())


@pytest.mark.gpu
def test_model_postprocess_api():
    """OmniVGGT.postprocess adds the keys inference.py computes on the host (extrinsic / intrinsic / unprojected points /
    confidence mask) and they agree with the oracle applied to the same predictions."""
    from test_model_gpu import model
    from oracle.synth import make_inputs
    m = model("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
    pred = m.postprocess(m(depth_gt_index=[1], camera_gt_index=[0], **inp), conf_percent=25.0)
    torch.cuda.synchronize()
    check_postprocess_against_oracle(pred, 25.0)


def check_postprocess_against_oracle(pred, pct):
    """The keys postprocess added to the predictions of one scene against the oracle on the same predictions."""
    H, W = pred["images"].shape[-2:]
    ext, intr = PO.pose_encoding_to_extri_intri(pred["pose_enc"].cpu().numpy(), H, W)
    assert np.allclose(pred["extrinsic"].cpu().numpy(), ext, rtol=1e-4, atol=1e-5)
    assert np.allclose(pred["intrinsic"].cpu().numpy(), intr, rtol=1e-4, atol=1e-3)
    world = PO.unproject_depth_map_to_point_map(pred["depth"][0, ..., 0].cpu().numpy(), ext[0], intr[0])
    got = pred["world_points_from_depth"][0].cpu().numpy()
    assert np.abs(got - world).max() <= 1e-4 * np.abs(world).max()
    mask, thr = PO.conf_percentile_mask(pred["depth_conf"].cpu().numpy(), pct)
    assert pred["conf_threshold"].item() == float(thr) or (np.isnan(thr) and np.isnan(pred["conf_threshold"].item()))
    assert np.array_equal(pred["conf_mask"].cpu().numpy(), mask) and pred["conf_mask"].shape == pred["depth_conf"].shape
