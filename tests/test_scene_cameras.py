"""Which cameras the scene functions use, for every set of camera keys a predictions dict can hold (pose_enc always there):
the E0 of point_cloud's and mesh's align, tracks' extrinsic / intrinsic, the tensors that reach ovg_unproject_depth and the
number of pose_enc decodes.  CPU dry run: the C library replaced by a recorder, ops.pose_decode by a counting fake whose
cameras are filled with constants of their own."""
import itertools

import pytest
import torch

from ovg_support import install

B, S, H, W = 2, 3, 4, 5
SCENE = 1
OWN, DECODED = 10.0, 20.0          # translations (plus the view index) of the predictions' and of the decoded extrinsics
OWN_K, DECODED_K, DECODED_C2W = 2.0, 3.0, 4.0
COMBOS = list(itertools.product((False, True), repeat=3))      # extrinsic, intrinsic, world_points_from_depth present


def _cameras(t, k):
    ext = torch.eye(4)[:3].repeat(S, 1, 1)
    ext[:, :, 3] = t + torch.arange(S, dtype=torch.float32)[:, None]
    return ext, torch.full((S, 3, 3), k)


def tracks_decodes(has_ext, has_intr, unproject):
    """pose_enc decodes of one tracks call: one whenever a camera is missing or the depth is unprojected."""
    return int(not (has_ext and has_intr) or unproject)


@pytest.fixture()
def dry(monkeypatch):
    from omnivggt_official_b200 import ops

    def read(t):                  # counts read zero; the fp64 reads of point_cloud and mesh carry E0 and read as they are
        return t.cpu() if t.dtype == torch.float64 else torch.zeros_like(t, device="cpu")

    def pose_decode(pose_enc, h, w):
        assert pose_enc.dtype == torch.float32 and tuple(pose_enc.shape) == (S, 9) and (h, w) == (H, W)
        assert (pose_enc == SCENE).all()
        cams = _cameras(DECODED, DECODED_K) + (torch.full((S, 3, 4), DECODED_C2W),)
        fake.decoded.append(cams)                               # kept alive: their pointers identify them
        return cams

    fake = install(monkeypatch, read=read, read_in_calls=False)
    fake.decoded = []
    monkeypatch.setattr(ops, "pose_decode", pose_decode)
    return fake


def _predictions(has_ext, has_intr, has_wpfd):
    g = torch.Generator().manual_seed(0)
    pred = {"images": torch.rand(B, S, 3, H, W, generator=g),
            "pose_enc": torch.arange(float(B))[:, None, None].repeat(1, S, 9),
            "depth": 1.0 + torch.rand(B, S, H, W, 1, generator=g), "depth_conf": 1.0 + torch.rand(B, S, H, W, generator=g),
            "world_points": torch.randn(B, S, H, W, 3, generator=g),
            "world_points_conf": 1.0 + torch.rand(B, S, H, W, generator=g)}
    ext, intr = _cameras(OWN, OWN_K)
    if has_ext:
        pred["extrinsic"] = torch.stack([torch.zeros_like(ext), ext])
    if has_intr:
        pred["intrinsic"] = torch.stack([torch.zeros_like(intr), intr])
    if has_wpfd:
        pred["world_points_from_depth"] = torch.randn(B, S, H, W, 3, generator=g)
    return pred


def _check_unprojection(dry, pred, unproject):
    calls = [a for n, a in dry.calls if n == "ovg_unproject_depth"]
    if not unproject:
        assert calls == []
        return
    (a,) = calls                                            # depth, intrinsic, cam2world, world, K, H, W, stream
    _, intr, c2w = dry.decoded[-1]
    assert a[0] == pred["depth"][SCENE].data_ptr() and a[1] == intr.data_ptr() and a[2] == c2w.data_ptr()
    assert a[4:7] == (S, H, W)


@pytest.mark.parametrize("source", ["depth", "pointmap"])
@pytest.mark.parametrize("has_ext,has_intr,has_wpfd", COMBOS)
def test_camera_rules(dry, has_ext, has_intr, has_wpfd, source):
    from omnivggt_official_b200 import OmniVGGT
    pred = _predictions(has_ext, has_intr, has_wpfd)
    unproject = source == "depth" and not has_wpfd
    own_ext, own_intr = _cameras(OWN, OWN_K)
    dec_ext, dec_intr = _cameras(DECODED, DECODED_K)
    # align's E0: the camera the points were made with -- decoded when the depth is unprojected, else the predictions' own
    e0_decoded = unproject or not has_ext
    for fn, frame in ((OmniVGGT.point_cloud, None), (OmniVGGT.mesh, 2)):
        dry.calls.clear(), dry.reads.clear(), dry.decoded.clear()
        fn(pred, source=source, scene=SCENE, frame=frame)
        assert len(dry.decoded) == int(e0_decoded)
        (host,) = dry.reads
        assert torch.equal(host[-12:].view(3, 4).float(), (dec_ext if e0_decoded else own_ext)[frame or 0]), fn.__name__
        _check_unprojection(dry, pred, unproject)
    # tracks: the predictions' extrinsic and intrinsic, each on its own, decoded where missing
    dry.calls.clear(), dry.reads.clear(), dry.decoded.clear()
    out = OmniVGGT.tracks(pred, source=source, scene=SCENE)
    assert len(dry.decoded) == tracks_decodes(has_ext, has_intr, unproject)
    assert torch.equal(out["extrinsic"], own_ext if has_ext else dec_ext)
    assert torch.equal(out["intrinsic"], own_intr if has_intr else dec_intr)
    _check_unprojection(dry, pred, unproject)


@pytest.mark.parametrize("has_ext,has_intr", [(False, False), (True, False), (False, True)])
def test_tracks_without_cameras_or_pose_enc_raises_before_any_device_work(dry, has_ext, has_intr):
    from omnivggt_official_b200 import OmniVGGT
    pred = _predictions(has_ext, has_intr, True)
    del pred["pose_enc"]
    with pytest.raises(ValueError, match="tracks need extrinsic and intrinsic, or pose_enc to decode them from"):
        OmniVGGT.tracks(pred, scene=SCENE)
    assert dry.calls == [] and dry.decoded == []
