"""Helpers shared by the test modules (pytest does not collect this module: its name does not start with test_).

FakeLibrary and install() stand in for libovg in the CPU dry runs: the package runs on CPU tensors and every entry point it
calls is recorded instead of launched.  install() is the one place that knows the seams through which the package reaches the
library and the host.  A module whose dry run needs other answers builds its own ``dry`` fixture on install()."""
import hashlib
import json
import struct

import numpy as np
import pytest
import torch

from conftest import golden_schema

F32 = torch.float32
GUARD = 4096                # elements in each sentinel band of guarded()


# ------------------------------------------------------------------------------------------------------------------ dry runs
class FakeLibrary:
    """libovg replaced by a recorder.  Every entry point is recorded as (name, args) in ``calls`` and returns 0 (OVG_OK), except
    ``*_workspace_bytes``, which answers ``workspace_bytes``.  ``*_create`` keeps a copy of its descriptor in ``descs``;
    ``effects[name](args)`` runs for an entry point whose output the caller goes on to use."""

    def __init__(self, workspace_bytes=0, effects=None):
        self.calls, self.reads, self.descs = [], [], {}
        self.workspace_bytes, self.effects = workspace_bytes, effects or {}

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            if name.endswith("_create"):
                d = a[0]._obj                       # ctypes.byref(desc)
                self.descs[name] = type(d).from_buffer_copy(d)
            if name in self.effects:
                self.effects[name](a)
            return self.workspace_bytes if name.endswith("_workspace_bytes") else 0
        return fn

    def names(self):
        return [n for n, _ in self.calls]

    def count(self, name):
        return sum(n == name for n, _ in self.calls)

    def args(self, name):
        return [a for n, a in self.calls if n == name]


def host_copy(t):
    return t.cpu()


def host_zeros(t):
    return torch.zeros_like(t, device="cpu")


def install(monkeypatch, read=host_copy, read_in_calls=True, **library):
    """Puts a FakeLibrary(**library) in place of libovg and its stream, lets CPU tensors pass as device tensors, and replaces
    ops.host_read: each read appends the tensor to ``fake.reads`` (and ("host_read", ()) to ``fake.calls`` if
    ``read_in_calls``) and returns read(tensor).  Returns the fake."""
    from omnivggt_official_b200 import _lib, ops
    fake = FakeLibrary(**library)

    def host_read(t):
        if read_in_calls:
            fake.calls.append(("host_read", ()))
        fake.reads.append(t)
        return read(t)

    monkeypatch.setattr(_lib, "lib", lambda: fake)
    monkeypatch.setattr(_lib, "stream", lambda: 0)
    monkeypatch.setattr(ops, "_on_device", lambda t: True)
    monkeypatch.setattr(ops, "host_read", host_read)
    return fake


@pytest.fixture()
def dry(monkeypatch):
    """libovg replaced by a FakeLibrary, on CPU tensors; host reads return the tensor and go into ``calls`` and ``reads``."""
    return install(monkeypatch)


@pytest.fixture(name="dry")
def dry_workspaces(monkeypatch):
    """``dry`` for the forward and the poisoning allocator: every workspace is a real buffer whose pointer can be checked
    (test_poison_cpu.py), and ``calls`` holds library calls only."""
    return install(monkeypatch, read_in_calls=False, workspace_bytes=4096)


def mini_model(variant="mini_conv"):
    from omnivggt_official_b200 import OmniVGGT
    v = golden_schema(variant)["variant"]
    kw = dict(img_size=v["img_size"], embed_dim=v["embed_dim"], depth=v["depth"], dpt_features=v["features"],
              dpt_out_channels=v["out_channels"], dpt_layers=tuple(range(v["depth"]))[-4:], camera_heads=v["cam_heads"],
              camera_trunk_depth=v["cam_trunk"])
    if v["patch_embed"] == "conv":
        kw.update(patch_embed="conv")
    else:
        kw.update(patch_embed="dino", dino_depth=2, dino_heads=2)
    return OmniVGGT(**kw)


def scene(S, H, W, seed=3, distinct_cameras=False):
    """Predictions of one scene on the host: random images, depth points and confidences, identity cameras (translated by the
    view index if ``distinct_cameras``)."""
    g = torch.Generator().manual_seed(seed)
    ext = torch.eye(4)[:3].repeat(1, S, 1, 1)
    if distinct_cameras:
        ext[0, :, :, 3] = torch.arange(S, dtype=torch.float32)[:, None]
    return {"images": torch.rand(1, S, 3, H, W, generator=g), "world_points_from_depth": torch.randn(1, S, H, W, 3, generator=g),
            "depth_conf": 1.0 + torch.rand(1, S, H, W, generator=g), "extrinsic": ext}


# ------------------------------------------------------------------------------------------------------------------ outputs
def sha256(a, hex=True):
    """SHA-256 of an array's bytes in C order: the hex string, or the raw digest if not ``hex``."""
    h = hashlib.sha256(np.ascontiguousarray(a).tobytes())
    return h.hexdigest() if hex else h.digest()


def parse_glb(data: bytes):
    """(JSON document, binary chunk) of a .glb file; the binary chunk is b"" when the file has none."""
    magic, version, total = struct.unpack_from("<III", data, 0)
    assert magic == 0x46546C67 and version == 2 and total == len(data)
    jlen, jtype = struct.unpack_from("<II", data, 12)
    assert jtype == 0x4E4F534A and jlen % 4 == 0
    doc = json.loads(data[20:20 + jlen].decode())
    off = 20 + jlen
    if off == total:
        return doc, b""
    blen, btype = struct.unpack_from("<II", data, off)
    assert btype == 0x004E4942 and blen % 4 == 0 and off + 8 + blen == total
    return doc, data[off + 8:off + 8 + blen]


# ------------------------------------------------------------------------------------------------------------------ GPU kernels
def ops_module():
    from omnivggt_official_b200 import ops
    return ops


def lib_module():
    from omnivggt_official_b200 import _lib
    return _lib


def rel(a, b, host=False):
    """Relative L2 error of a against b, in fp32 (on the host if ``host``)."""
    a, b = a.float(), b.float()
    if host:
        a, b = a.cpu(), b.cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def randn(*s, scale=1.0, seed=0, dtype=F32, host_rng=False):
    """Seeded normal samples times ``scale`` on the GPU, as ``dtype``; drawn by a host generator if ``host_rng``."""
    g = torch.Generator(device="cpu" if host_rng else "cuda").manual_seed(seed)
    return (torch.randn(*s, generator=g, device=g.device) * scale).to("cuda", dtype)


def margin(name, r):
    print(f"margin {name}: {r:.3f}")


def guarded(n, dtype, fill):
    """A flat buffer with `n` elements between two sentinel guards: (buffer, the n-element middle)."""
    buf = torch.full((GUARD + n + GUARD,), fill, device="cuda", dtype=dtype)
    return buf, buf[GUARD:GUARD + n]


def guards_ok(buf, fill):
    ref = torch.full((GUARD,), fill, device="cuda", dtype=buf.dtype)
    return torch.equal(buf[:GUARD], ref) and torch.equal(buf[-GUARD:], ref)
