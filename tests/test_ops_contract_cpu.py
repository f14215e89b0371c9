"""Operand contracts at the libovg boundary (CPU dry runs): every malformed operand a wrapper hands to the library as a raw
pointer is refused with TypeError (dtype, device) or ValueError (shape, size, layout) before any library call, also under
``python -O``; a size query that rejects its arguments raises OvgError before any compute entry point.

Each case starts from well-formed operands of one wrapper (BASES) and breaks one of them; ``off`` marks a tensor that
ops._on_device refuses."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from omnivggt_official_b200 import _lib as L, ops, preprocess
from ovg_support import install, mini_model

F32, F64, BF16, U8, I32, I64 = torch.float32, torch.float64, torch.bfloat16, torch.uint8, torch.int32, torch.int64
TESTS = os.path.dirname(os.path.abspath(__file__))


def z(*shape, dtype=F32):
    return torch.zeros(*shape, dtype=dtype)


# ------------------------------------------------------------------------------------------------------------------ mutations
_OFF = set()


def off(t):
    """t itself, refused by ops._on_device."""
    _OFF.add(id(t))
    return t


def strided(t):
    """A non-contiguous view of t's shape and dtype, with stride 2 in the last dim."""
    return torch.zeros(*t.shape[:-1], 2 * t.shape[-1], dtype=t.dtype)[..., ::2]


def dtype(d):
    return "dtype", lambda t: t.to(d), TypeError


def size(*shape):
    return "size", lambda t: torch.zeros(*shape, dtype=t.dtype), ValueError


OFF = ("device", off, TypeError)
STRIDED = ("strided", strided, ValueError)


# ------------------------------------------------------------------------------------------------------------------ bases
BASES = {}


def base(make):
    """make() -> (call, operands): call(**operands) is a well-formed call of one wrapper."""
    BASES[make.__name__] = make
    return make


@base
def gemm():
    return (lambda a, b, epi, out: ops.gemm(a, b, epi=epi, out=out, ldo=out.stride(0)),
            dict(a=z(8, 16, dtype=BF16), b=z(4, 16, dtype=BF16), epi=L.EPI_BF16, out=z(8, 4, dtype=BF16)))


@base
def linear_resid():
    return ops.linear_resid, dict(a=z(8, 16, dtype=BF16), w=z(4, 16, dtype=BF16), bias=z(4), gamma=z(4), x=z(8, 4))


@base
def attention():
    return (lambda q, k, v, out: ops.attention(q, k, v, out, 1, 1, 4),
            dict(q=z(1, 1, 4, 64, dtype=BF16), k=z(1, 1, 4, 64, dtype=BF16), v=z(1, 1, 4, 64, dtype=BF16),
                 out=z(1, 4, 64, dtype=BF16)))


@base
def attention_scratch():
    return ops.attention_scratch, dict(device="cpu")


@base
def layernorm():
    return ops.layernorm, dict(x=z(4, 8), out=z(4, 8))


@base
def upsample_bilinear():
    return (lambda src, dst: ops.upsample_bilinear(src, dst, None, None, 1, 2, 2, 4, 4, 8),
            dict(src=z(1, 2, 2, 8, dtype=BF16), dst=z(1, 4, 4, 8, dtype=BF16)))


@base
def dpt_tail():
    return (lambda src, w3x3: ops.dpt_tail(src, None, None, w3x3, z(32), z(2, 32), z(2), 0, 1, 2, 2, 4, 4),
            dict(src=z(1, 4, 4, 128, dtype=BF16), w3x3=z(32, 9 * 128, dtype=BF16)))


@base
def pose_decode():
    return ops.pose_decode, dict(pose_enc=z(2, 9), H=4, W=4)


@base
def unproject_depth():
    return ops.unproject_depth, dict(depth=z(2, 4, 4), intrinsic=z(2, 3, 3), cam2world=z(2, 3, 4), H=4, W=4)


@base
def conf_percentile_mask():
    return ops.conf_percentile_mask, dict(conf=z(2, 4, 4), percent=50.0)


@base
def point_cloud_workspace():
    return ops.point_cloud_workspace, dict(n=32, device="cpu")


@base
def point_cloud_count():
    return ops.point_cloud_count, dict(conf_mask=z(2, 4, 4, dtype=U8), images=z(2, 3, 4, 4), ws=z(0, dtype=U8))


@base
def point_cloud_gather():
    return (ops.point_cloud_gather,
            dict(points=z(2, 4, 4, 3), conf_mask=z(2, 4, 4, dtype=U8), images=z(2, 3, 4, 4), ws=z(0, dtype=U8), n_kept=3))


@base
def point_cloud_center():
    return ops.point_cloud_center, dict(points=z(5, 3), ws=z(0, dtype=U8))


@base
def point_cloud_scale():
    return ops.point_cloud_scale, dict(xyz=z(3, 8), n_kept=5, ws=z(0, dtype=U8))


@base
def segment_sky():
    return (lambda image, conf: ops.segment_sky(image, 2, 4, 4, 48, 3, 1, conf),
            dict(image=z(2, 4, 4, 3, dtype=U8), conf=z(2, 4, 4)))


@base
def sky_mask_conf():
    return ops.sky_mask_conf, dict(conf=z(8), sky=z(8, dtype=U8))


@base
def farthest_point_sample():
    return ops.farthest_point_sample, dict(xyz=z(2, 8, 3), npoint=4, start=z(2, dtype=I64))


@base
def compute_ranking():
    return ops.compute_ranking, dict(ext=z(4, 3, 4), lambda_t=1.0, normalize=True, out_dtype=F32, k=2)


@base
def sim3_estimate():
    return ops.sim3_estimate, dict(src=z(8, 3), dst=z(8, 3), keep=z(8, dtype=U8))


@base
def sim3_apply():
    def call(sim3, p_in, p_out, d_in, d_out, e_in, e_out, pairs):
        ops.sim3_apply(sim3, 2, 4, points=((p_in, p_out),) * pairs, depth=(d_in, d_out), ext=(e_in, e_out))
    return call, dict(sim3=z(4, 4, dtype=F64), p_in=z(8, 3), p_out=z(8, 3), d_in=z(8), d_out=z(8), e_in=z(2, 3, 4),
                      e_out=z(2, 3, 4), pairs=1)


@base
def bundle_adjust():
    def call(**operands):
        return ops.bundle_adjust(**operands, iterations=2, refine_focal=True, loss="cauchy", loss_scale=1.0)
    return call, dict(points=z(3, 3, dtype=F64), offsets=z(4, dtype=I64), view=z(6, dtype=I32),
                      observations=z(6, 2, dtype=F64), extrinsic=z(2, 3, 4), intrinsic=z(2, 3, 3))


@base
def Mesher():
    return ops.Mesher, dict(keep=z(32, dtype=U8), images=z(2, 3, 4, 4), F=2, H=4, W=4)


@base
def Mesher_faces():
    mesher = ops.Mesher(z(32, dtype=U8), z(2, 3, 4, 4), 2, 4, 4)
    return (lambda colors: mesher.faces(3, colors)), dict(colors=z(32, 3))


@base
def Mesher_compact():
    meshers = {True: ops.Mesher(z(32, dtype=U8), z(2, 3, 4, 4), 2, 4, 4), False: ops.Mesher(z(32, dtype=U8), None, 2, 4, 4)}
    return (lambda points, images: meshers[images].compact(points, 3, 2)), dict(points=z(2, 4, 4, 3), images=True)


@base
def Matcher():
    return ops.Matcher, dict(points=z(2, 16, 3), keep=z(32, dtype=U8), pairs=z(1, 2, dtype=I32))


@base
def Tracker():
    return ops.Tracker, dict(matcher=ops.Matcher(z(2, 16, 3), None, z(1, 2, dtype=I32)), pair_off=z(3, dtype=I32), min_views=2)


@base
def Tracker_gather():
    tracker = ops.Tracker(ops.Matcher(z(2, 16, 3), None, z(1, 2, dtype=I32)), z(3, dtype=I32), 2)
    return ((lambda images, extrinsic, intrinsic: tracker.gather(images, extrinsic, intrinsic, 4, 3, 6)),
            dict(images=z(2, 3, 4, 4), extrinsic=z(2, 3, 4), intrinsic=z(2, 3, 3)))


_ENGINE = []


@base
def Engine_aggregate():
    """mini_conv: 4 layers of [K, T, 2C] = [2, 9, 256] for two 28 x 28 views."""
    from omnivggt_official_b200.engine import Engine
    if not _ENGINE:
        _ENGINE.append(Engine(mini_model().eval()))
    eng = _ENGINE[0]

    def call(keep, cp, B, layers):
        eng.aggregate(z(1), z(1), None, None, [], B, 2 // B, 28, 28, keep, cp=cp, views_total=2, slots=False, layers=layers)
    return call, dict(keep=eng.keep, cp=None, B=1, layers=[z(2 * 9 * 256) for _ in range(eng.depth)])


@base
def resize_view():
    return (lambda im: preprocess._resize_view(L.lib(), 0, im, 8, 6, 0, 6, z(3, 6, 8), "cpu")), dict(im=np.zeros((6, 8, 3), np.uint8))


# ------------------------------------------------------------------------------------------------------------------ cases
def each(name, operand, *kinds):
    return [(f"{name}-{operand}-{label}", name, {operand: mutate}, exc) for label, mutate, exc in kinds]


def const(label, value, exc=ValueError):
    return label, lambda _: value, exc


def layer(kind):
    """A kind applied to layers[1]."""
    label, mutate, exc = kind
    return label, lambda ls: [ls[0], mutate(ls[1]), *ls[2:]], exc


CASES = [
    *each("gemm", "a", dtype(F32), OFF, size(16), STRIDED),
    *each("gemm", "b", dtype(torch.float16), OFF, size(4, 15), size(4, 16, 1), STRIDED),
    *each("gemm", "out", OFF, STRIDED),
    ("gemm-f16-epi", "gemm", {"a": lambda t: t.half(), "b": lambda t: t.half(), "epi": lambda _: L.EPI_RESID}, ValueError),
    *each("linear_resid", "x", dtype(BF16), OFF),
    *[c for o in ("q", "k", "v", "out") for c in each("attention", o, dtype(F32), OFF, STRIDED)],
    *each("layernorm", "x", dtype(torch.float16), OFF, STRIDED),
    *each("layernorm", "out", dtype(F64), OFF, STRIDED),
    *each("upsample_bilinear", "src", dtype(F32), OFF),
    *each("upsample_bilinear", "dst", dtype(torch.float16), OFF),
    *each("dpt_tail", "src", dtype(F32), OFF, STRIDED),
    *each("dpt_tail", "w3x3", dtype(torch.float16), OFF, STRIDED),
    *each("pose_decode", "pose_enc", dtype(F64), OFF),
    *each("unproject_depth", "depth", dtype(F64), OFF),
    *each("unproject_depth", "intrinsic", dtype(F64), OFF, size(1, 3, 3)),
    *each("unproject_depth", "cam2world", dtype(F64), OFF, size(2, 3, 3)),
    *each("conf_percentile_mask", "conf", dtype(F64), OFF),
    *each("point_cloud_count", "conf_mask", dtype(torch.bool), OFF, size(2, 4, 3), STRIDED),
    *each("point_cloud_count", "images", dtype(F64), OFF, size(2, 4, 4, 4), STRIDED),
    *each("point_cloud_gather", "points", dtype(F64), OFF, size(5, 3), STRIDED),
    *each("point_cloud_gather", "conf_mask", dtype(torch.bool), OFF, size(2, 4, 3), STRIDED),
    *each("point_cloud_gather", "images", dtype(F64), OFF, size(2, 4, 4, 4), STRIDED),
    *each("point_cloud_center", "points", dtype(F64), OFF, STRIDED),
    *each("point_cloud_scale", "xyz", dtype(F64), OFF),
    *each("segment_sky", "image", dtype(F64), OFF),
    *each("segment_sky", "conf", dtype(F64), OFF, size(2, 4, 3), STRIDED),
    *each("sky_mask_conf", "conf", dtype(F64), OFF, STRIDED),
    *each("sky_mask_conf", "sky", dtype(F32), OFF, size(7), STRIDED),
    *each("farthest_point_sample", "xyz", dtype(F64), OFF, size(2, 8, 2), STRIDED),
    *each("farthest_point_sample", "start", dtype(I32), OFF, size(3), STRIDED),
    *each("compute_ranking", "ext", dtype(torch.float16), OFF, size(4, 2, 4), size(4, 3, 3), size(4, 12)),
    *each("compute_ranking", "out_dtype", const("value", torch.float16)),
    *each("sim3_estimate", "src", dtype(F64), OFF, size(8, 2), STRIDED),
    *each("sim3_estimate", "dst", dtype(F64), OFF, size(7, 3), STRIDED),
    *each("sim3_estimate", "keep", dtype(torch.bool), OFF, size(7), STRIDED),
    *each("sim3_apply", "sim3", dtype(F32), OFF, size(3, 4), STRIDED),
    *[c for o in ("p_in", "p_out", "d_in", "d_out", "e_in", "e_out") for c in each("sim3_apply", o, dtype(F64), OFF, size(5), STRIDED)],
    *each("sim3_apply", "pairs", const("three", 3)),
    *each("bundle_adjust", "points", dtype(F32), OFF, size(3, 2), STRIDED),
    *each("bundle_adjust", "offsets", dtype(I32), OFF, size(5), STRIDED),
    *each("bundle_adjust", "view", dtype(I64), OFF, size(6, 1), STRIDED),
    *each("bundle_adjust", "observations", dtype(F32), OFF, size(6, 3), STRIDED),
    *each("bundle_adjust", "extrinsic", dtype(F64), OFF, size(2, 4, 4), STRIDED),
    *each("bundle_adjust", "intrinsic", dtype(F64), OFF, size(2, 3, 4), STRIDED),
    *each("Mesher", "keep", dtype(torch.bool), OFF, size(31), STRIDED),
    *each("Mesher", "images", dtype(F64), OFF, size(2, 3, 4, 5), STRIDED),
    *each("Mesher_faces", "colors", OFF, size(31, 3), STRIDED),
    *each("Mesher_compact", "points", dtype(F64), OFF, size(2, 4, 4, 2), STRIDED),
    *each("Mesher_compact", "images", const("none", False)),
    *each("Matcher", "points", dtype(F64), OFF, size(2, 16, 2), STRIDED),
    *each("Matcher", "keep", dtype(torch.bool), OFF, size(31), STRIDED),
    *each("Matcher", "pairs", dtype(I64), OFF, STRIDED),
    *each("Tracker", "pair_off", dtype(I64), OFF, size(2), STRIDED),
    *each("Tracker_gather", "images", dtype(F64), OFF, size(2, 3, 8, 2), STRIDED),
    *each("Tracker_gather", "extrinsic", dtype(F64), OFF, size(2, 3, 3), STRIDED),
    *each("Tracker_gather", "intrinsic", dtype(F64), OFF, size(2, 4, 3), STRIDED),
    *each("Engine_aggregate", "keep", const("other", (0, 1))),
    ("Engine_aggregate-cp-B2", "Engine_aggregate", {"cp": lambda _: object(), "B": lambda _: 2, "layers": lambda _: None},
     ValueError),
    *each("Engine_aggregate", "cp", const("with-layers", object())),
    *each("Engine_aggregate", "layers", const("count", [z(2 * 9 * 256)] * 3),
          *[layer(k) for k in (dtype(F64), OFF, size(2 * 9 * 256 - 1), STRIDED)]),
    *each("resize_view", "im", const("gray-array", np.zeros((6, 8), np.uint8)), const("gray-tensor", z(6, 8, dtype=U8)),
          const("rgba", np.zeros((6, 8, 4), np.uint8))),
]

# the wrappers that size a workspace with a *_workspace_bytes query
QUERIES = ["point_cloud_workspace", "segment_sky", "farthest_point_sample", "compute_ranking", "sim3_estimate", "bundle_adjust",
           "Mesher", "Matcher", "Tracker"]


def outcome(monkeypatch, name, changes):
    """(exception name or None, library calls of the call) of BASES[name] with ``changes`` applied to its operands."""
    fake = install(monkeypatch)
    _OFF.clear()
    monkeypatch.setattr(ops, "_on_device", lambda t: id(t) not in _OFF)
    call, operands = BASES[name]()
    fake.calls.clear()
    try:
        call(**dict(operands, **{k: mutate(operands[k]) for k, mutate in changes.items()}))
    except Exception as e:      # noqa: BLE001  (the exception type is the result)
        return type(e).__name__, fake.names()
    return None, fake.names()


def outcomes():
    """{case id: [exception name, library calls]} of every case."""
    with pytest.MonkeyPatch.context() as mp:
        return {cid: list(outcome(mp, name, changes)) for cid, name, changes, _ in CASES}


# ------------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name", sorted(BASES))
def test_well_formed_operands_reach_the_library(monkeypatch, name):
    err, calls = outcome(monkeypatch, name, {})
    assert err is None and calls


def test_every_contract_is_covered():
    assert {name for _, name, _, _ in CASES} == set(BASES) - {"attention_scratch", "point_cloud_workspace"}


@pytest.mark.parametrize("cid,name,changes,exc", CASES, ids=[c[0] for c in CASES])
def test_malformed_operand_is_refused(monkeypatch, cid, name, changes, exc):
    assert outcome(monkeypatch, name, changes) == (exc.__name__, [])


def test_refused_under_python_O():
    """The same table in an interpreter that strips assert statements."""
    driver = ("import json, sys\n"
              f"sys.path[:0] = [{os.path.dirname(TESTS)!r}, {TESTS!r}]\n"
              "assert False, 'asserts are live'\n"
              "import test_ops_contract_cpu as t\n"
              "print(json.dumps(t.outcomes()))\n")
    flags = ["-O"] + (["-s"] if sys.flags.no_user_site else [])
    out = subprocess.run([sys.executable, *flags, "-c", driver], capture_output=True, text=True, timeout=600, cwd=TESTS)
    assert out.returncode == 0, out.stderr[-3000:]
    got = json.loads(out.stdout.strip().splitlines()[-1])
    assert got == {cid: [exc.__name__, []] for cid, _, _, exc in CASES}


@pytest.mark.parametrize("name", QUERIES)
def test_failed_size_query_raises_before_compute(monkeypatch, name):
    fake = install(monkeypatch)
    call, operands = BASES[name]()
    fake.workspace_bytes = -1
    fake.calls.clear()
    with pytest.raises(L.OvgError, match="_workspace_bytes"):
        call(**operands)
    assert len(fake.calls) == 1 and fake.calls[0][0].endswith("_workspace_bytes")


def test_failed_size_query_stops_the_forward(monkeypatch):
    from oracle.synth import make_inputs
    from omnivggt_official_b200.engine import Engine
    fake = install(monkeypatch, read_in_calls=False, workspace_bytes=-1)
    m = mini_model().eval()
    m._engine = Engine(m)
    with pytest.raises(L.OvgError, match="ovg_aggregator_workspace_bytes"):
        m(**make_inputs(1, 2, 28, 28, seed=1))
    assert fake.names() and all(n.endswith(("_create", "_workspace_bytes")) for n in fake.names())
