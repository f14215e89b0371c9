"""CPU tests (no GPU): C-ABI library loads and exports every declared symbol, ctypes struct layout matches the C
header, parameter schema equals the reference checkpoint schema, host-side PyTorch parts agree with the oracle, and the
product refuses to run without a CUDA device (no CPU fallback)."""
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch

from conftest import GOLDEN, ROOT, golden_index, golden_schema
from oracle import omnivggt_oracle as O
from oracle.synth import make_inputs, make_state_dict
from ovg_support import mini_model


def test_library_exports_every_declared_symbol_at_abi_version_5():
    from omnivggt_official_b200 import _lib
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "ovg.h")).read()
    declared = set(re.findall(r"\b(ovg_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/ovg.h but not exported by libovg.so"
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    assert lib.ovg_version() == 5


def test_ctypes_struct_matches_header():
    from omnivggt_official_b200 import _lib
    fields = [f[0] for f in _lib.GemmArgs._fields_]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"ovg.h\"\nint main(){printf(\"%zu\\n\", sizeof(ovg_gemm_args));\n"
    for f in fields:
        src += f'printf("%zu\\n", offsetof(ovg_gemm_args, {f}));\n'
    src += "return 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        out = subprocess.check_output([os.path.join(d, "t")]).decode().split()
    assert int(out[0]) == ctypes.sizeof(_lib.GemmArgs)
    for f, off in zip(fields, out[1:]):
        assert getattr(_lib.GemmArgs, f).offset == int(off), f


@pytest.mark.parametrize("cname,pyname", [("ovg_block_weights", "BlockWeights"), ("ovg_aggregator_desc", "AggregatorDesc"),
                                          ("ovg_dino_desc", "DinoDesc"), ("ovg_dpt_fusion", "DptFusion"), ("ovg_dpt_desc", "DptDesc"),
                                          ("ovg_camera_desc", "CameraDesc")])
def test_runtime_structs_match_header(cname, pyname):
    from omnivggt_official_b200 import _lib
    cls = getattr(_lib, pyname)
    fields = [f[0] for f in cls._fields_]
    src = f"#include <stdio.h>\n#include <stddef.h>\n#include \"ovg.h\"\nint main(){{printf(\"%zu\\n\", sizeof({cname}));\n"
    for f in fields:
        src += f'printf("%zu\\n", offsetof({cname}, {f}));\n'
    src += "return 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        out = subprocess.check_output([os.path.join(d, "t")]).decode().split()
    assert int(out[0]) == ctypes.sizeof(cls)
    for f, off in zip(fields, out[1:]):
        assert getattr(cls, f).offset == int(off), f


@pytest.mark.parametrize("variant", ["mini_conv", "mini_dino"])
def test_state_dict_schema_equals_reference(variant):
    m = mini_model(variant)
    schema = golden_schema(variant)["schema"]
    sd = m.state_dict()
    assert set(sd) == set(schema)
    for k, shp in schema.items():
        assert list(sd[k].shape) == shp, k
    m.load_state_dict(make_state_dict(schema, 0), strict=True)


def test_full_model_schema_size():
    from omnivggt_official_b200 import OmniVGGT
    with torch.device("meta"):
        m = OmniVGGT(init_seed=None)
    sd = m.state_dict()
    assert len(sd) == 1505                                   # SURVEY.md quick facts [probe]
    assert abs(sum(p.numel() for p in m.parameters()) / 1e6 - 1217.5) < 0.1
    assert "aggregator.patch_embed.blocks.23.ls2.gamma" in sd and "depth_head.scratch.output_conv2.2.bias" in sd


def test_no_cpu_fallback():
    m = mini_model()
    inp = make_inputs(1, 2, 56, 56, seed=1)
    with pytest.raises(RuntimeError):
        m(images=inp["images"])


def test_pose_encoding_and_injection_match_oracle():
    from omnivggt_official_b200 import torch_parts as TP
    m = mini_model()
    schema = golden_schema("mini_conv")["schema"]
    sd = make_state_dict(schema, 0)
    m.load_state_dict(sd)
    B, S, H, W = 2, 4, 56, 70
    inp = make_inputs(B, S, H, W, seed=3)
    idx = [0, 2, 3]
    ti = torch.tensor(idx)
    pose = TP.aux_pose_encoding(inp["extrinsics"][:, ti], inp["intrinsics"][:, ti], H, W)
    ref = O.pose_encoding(O.normalize_extrinsics(inp["extrinsics"][:, ti]), inp["intrinsics"][:, ti], H, W)
    assert torch.allclose(pose, ref, atol=1e-5)
    inj = TP.injection_vectors(TP.pack_injection(m.aggregator), pose, idx, B, S)
    C = 128
    rows = (torch.arange(B)[:, None] * S + ti[None]).reshape(-1)
    for layer in (0, 1, 4):
        g = torch.zeros(B * S, C)
        g[rows] = O.linear(ref, sd, f"aggregator.pose_embeddings.{layer}").reshape(-1, C)
        want = O.linear(g, sd, f"aggregator.camera_adapters.{layer}")
        assert torch.allclose(inj[layer], want, atol=1e-4), layer
    # no cameras: bias only, on every frame
    inj0 = TP.injection_vectors(TP.pack_injection(m.aggregator), None, [], B, S)
    assert torch.allclose(inj0[2], sd["aggregator.camera_adapters.2.bias"].expand(B * S, -1))
    # single selected camera: no scale normalisation (omnivggt_aggregator.py:98)
    p1 = TP.aux_pose_encoding(inp["extrinsics"][:, :1], inp["intrinsics"][:, :1], H, W)
    r1 = O.pose_encoding(O.normalize_extrinsics(inp["extrinsics"][:, :1]), inp["intrinsics"][:, :1], H, W)
    assert torch.allclose(p1, r1, atol=1e-5)


def test_uv_table_matches_oracle():
    from omnivggt_official_b200 import torch_parts as TP
    for C, h, w, a in ((64, 4, 4, 1.0), (128, 3, 5, 70 / 42), (32, 42, 70, 70 / 42)):
        t = TP.uv_posembed_table(C, h, w, a, "cpu")
        ref = O.uv_posembed(C, h, w, a).permute(1, 2, 0).reshape(h * w, C)
        assert torch.allclose(t, ref, atol=1e-6)
        tx, ty = TP.uv_posembed_separable(C, h, w, a, "cpu")
        sep = torch.cat([tx[None].expand(h, w, C // 2), ty[:, None].expand(h, w, C // 2)], -1).reshape(h * w, C)
        assert torch.allclose(sep, ref, atol=1e-6)


def test_dino_and_camera_head_match_oracle():
    from omnivggt_official_b200 import torch_parts as TP
    m = mini_model("mini_dino")
    meta = golden_schema("mini_dino")
    sd = make_state_dict(meta["schema"], 0)
    m.load_state_dict(sd)
    cfg = O.OracleConfig(dino_heads=2, camera_head_heads=meta["variant"]["cam_heads"])
    for H, W in ((56, 56), (42, 70)):
        img = torch.randn(2, 3, H, W)
        got = TP.dino_patchify(m.aggregator.patch_embed, img, 14, torch.float32)
        want = O.dino_patchify(sd, "aggregator.patch_embed", img, cfg)
        assert torch.allclose(got, want, atol=2e-4), (H, W)
    tok = torch.randn(2, 3, 1, 256)
    got = TP.camera_head(m.camera_head, tok[:, :, 0])
    want = O.camera_head(sd, "camera_head", tok, cfg)
    for a, b in zip(got, want):
        assert torch.allclose(a, b, atol=2e-4)
