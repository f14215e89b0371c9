"""glTF 2.0 binary (.glb) export of a point cloud from ``OmniVGGT.point_cloud`` -- the point-cloud part of the reference's
``--save_glb`` (inference.py:368-384 -> visual_util.py:238-267 trimesh.Scene.export) -- and of a triangle mesh from
``OmniVGGT.mesh(..., layout="glb")`` (``mesh_glb_bytes`` / ``write_mesh_glb``).  Host-only, numpy + the standard library.

    cloud = model.point_cloud(model.postprocess(predictions), conf_percent=0.0)
    write_glb("scene.glb", cloud)

One POINTS primitive with POSITION (float32 VEC3, with the min / max the specification requires) and COLOR_0 (normalised uint8
RGBA, alpha 255, so that every vertex attribute element is 4-byte aligned); ``cloud["align"]`` is the node matrix.  An empty
cloud is written as the reference's placeholder: one white point at (1, 0, 0) (visual_util.py:226-229).  The camera frustum
meshes of the reference are not written.
"""
from __future__ import annotations

import json
import struct

import numpy as np

GLB_MAGIC = 0x46546C67          # "glTF"
CHUNK_JSON = 0x4E4F534A         # "JSON"
CHUNK_BIN = 0x004E4942          # "BIN\0"
FLOAT, UNSIGNED_BYTE, UNSIGNED_INT, ARRAY_BUFFER, ELEMENT_ARRAY_BUFFER = 5126, 5121, 5125, 34962, 34963
POINTS, TRIANGLES = 0, 4


def _numpy(t) -> np.ndarray:
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def _container(doc: dict, binary: bytes) -> bytes:
    """The GLB container: header, the JSON chunk, and the BIN chunk when there is binary data."""
    js = json.dumps(doc, separators=(",", ":")).encode()
    js += b" " * (-len(js) % 4)                           # chunks are padded to 4 bytes: JSON with spaces, BIN with zeros
    binary += b"\0" * (-len(binary) % 4)
    chunks = struct.pack("<II", len(js), CHUNK_JSON) + js
    if binary:
        chunks += struct.pack("<II", len(binary), CHUNK_BIN) + binary
    return struct.pack("<III", GLB_MAGIC, 2, 12 + len(chunks)) + chunks


def _node(obj: dict) -> dict:
    node = {"mesh": 0}
    if obj.get("align") is not None:
        m = np.asarray(_numpy(obj["align"]), dtype=np.float64).reshape(4, 4)
        node["matrix"] = [float(v) for v in m.T.reshape(-1)]             # column-major
    return node


def glb_bytes(cloud: dict) -> bytes:
    """The .glb file of ``cloud`` (keys ``points`` [n,3], ``colors`` uint8 [n,3], optional ``align`` [4,4]) as bytes."""
    pts = np.ascontiguousarray(_numpy(cloud["points"]), dtype=np.float32).reshape(-1, 3)
    cols = np.ascontiguousarray(_numpy(cloud["colors"]), dtype=np.uint8).reshape(-1, 3)
    if len(pts) != len(cols):
        raise ValueError(f"{len(pts)} points but {len(cols)} colours")
    if len(pts) == 0:
        pts = np.array([[1.0, 0.0, 0.0]], dtype=np.float32)
        cols = np.array([[255, 255, 255]], dtype=np.uint8)
    n = len(pts)
    rgba = np.empty((n, 4), dtype=np.uint8)
    rgba[:, :3] = cols
    rgba[:, 3] = 255
    binary = pts.tobytes() + rgba.tobytes()             # 12 n + 4 n bytes: both views start 4-byte aligned
    node = _node(cloud)
    doc = {
        "asset": {"version": "2.0", "generator": "omnivggt_official_b200.glb"},
        "scene": 0,
        "scenes": [{"nodes": [0]}],
        "nodes": [node],
        "meshes": [{"primitives": [{"attributes": {"POSITION": 0, "COLOR_0": 1}, "mode": POINTS}]}],
        "buffers": [{"byteLength": len(binary)}],
        "bufferViews": [{"buffer": 0, "byteOffset": 0, "byteLength": 12 * n, "target": ARRAY_BUFFER},
                        {"buffer": 0, "byteOffset": 12 * n, "byteLength": 4 * n, "target": ARRAY_BUFFER}],
        "accessors": [{"bufferView": 0, "componentType": FLOAT, "count": n, "type": "VEC3",
                       "min": [float(v) for v in pts.min(0)], "max": [float(v) for v in pts.max(0)]},
                      {"bufferView": 1, "componentType": UNSIGNED_BYTE, "normalized": True, "count": n, "type": "VEC4"}],
    }
    return _container(doc, binary)


def write_glb(path: str, cloud: dict) -> None:
    """Write ``cloud`` (``OmniVGGT.point_cloud`` output) to ``path`` as a glTF 2.0 binary file."""
    data = glb_bytes(cloud)
    with open(path, "wb") as f:
        f.write(data)


def mesh_glb_bytes(mesh: dict) -> bytes:
    """The .glb file of a triangle mesh in the GLB layout of ``OmniVGGT.mesh(..., layout="glb")`` (keys ``positions`` fp32
    [m,3], ``colors`` uint8 [m,3], ``indices`` [k,3] into the positions, optional ``align`` [4,4]) as bytes.

    One TRIANGLES primitive: POSITION (float32 VEC3 with min / max), COLOR_0 (normalised uint8 RGBA, alpha 255) and uint32
    indices on an ELEMENT_ARRAY_BUFFER view, under a double-sided material, which shows both sides of every face as the
    reference's reversed duplicate faces do (viz.py:55,:57).  glTF has no per-face colour, so the file carries vertex colours:
    each vertex has its own pixel's colour, where the reference colours a face by one of its corners.  A mesh with no faces
    is a valid file with an empty scene.  Non-finite positions raise ValueError: glTF requires finite bounds."""
    pos = np.ascontiguousarray(_numpy(mesh["positions"]), dtype=np.float32).reshape(-1, 3)
    cols = np.ascontiguousarray(_numpy(mesh["colors"]), dtype=np.uint8).reshape(-1, 3)
    idx = np.ascontiguousarray(_numpy(mesh["indices"])).reshape(-1, 3)
    m, k = len(pos), len(idx)
    if len(cols) != m:
        raise ValueError(f"{m} positions but {len(cols)} colours")
    if k and (idx.min() < 0 or idx.max() >= m):
        raise ValueError("indices must be in [0, number of positions)")
    if not np.isfinite(pos).all():
        raise ValueError("mesh positions must be finite: glTF requires finite POSITION bounds")
    doc = {"asset": {"version": "2.0", "generator": "omnivggt_official_b200.glb"}, "scene": 0}
    if k == 0:
        doc["scenes"] = [{}]
        return _container(doc, b"")
    rgba = np.empty((m, 4), dtype=np.uint8)
    rgba[:, :3] = cols
    rgba[:, 3] = 255
    binary = pos.tobytes() + rgba.tobytes() + idx.astype(np.uint32).tobytes()   # 12 m + 4 m + 12 k: 4-byte aligned views
    doc.update({
        "scenes": [{"nodes": [0]}],
        "nodes": [_node(mesh)],
        "materials": [{"doubleSided": True, "pbrMetallicRoughness": {"metallicFactor": 0.0}}],
        "meshes": [{"primitives": [{"attributes": {"POSITION": 0, "COLOR_0": 1}, "indices": 2, "material": 0,
                                    "mode": TRIANGLES}]}],
        "buffers": [{"byteLength": len(binary)}],
        "bufferViews": [{"buffer": 0, "byteOffset": 0, "byteLength": 12 * m, "target": ARRAY_BUFFER},
                        {"buffer": 0, "byteOffset": 12 * m, "byteLength": 4 * m, "target": ARRAY_BUFFER},
                        {"buffer": 0, "byteOffset": 16 * m, "byteLength": 12 * k, "target": ELEMENT_ARRAY_BUFFER}],
        "accessors": [{"bufferView": 0, "componentType": FLOAT, "count": m, "type": "VEC3",
                       "min": [float(v) for v in pos.min(0)], "max": [float(v) for v in pos.max(0)]},
                      {"bufferView": 1, "componentType": UNSIGNED_BYTE, "normalized": True, "count": m, "type": "VEC4"},
                      {"bufferView": 2, "componentType": UNSIGNED_INT, "count": 3 * k, "type": "SCALAR"}],
    })
    return _container(doc, binary)


def write_mesh_glb(path: str, mesh: dict) -> None:
    """Write ``mesh`` (``OmniVGGT.mesh(..., layout="glb")`` output) to ``path`` as a glTF 2.0 binary file."""
    data = mesh_glb_bytes(mesh)
    with open(path, "wb") as f:
        f.write(data)
