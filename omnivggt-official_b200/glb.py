"""glTF 2.0 binary (.glb) export of a point cloud from ``OmniVGGT.point_cloud`` -- the point-cloud part of the reference's
``--save_glb`` (inference.py:368-384 -> visual_util.py:238-267 trimesh.Scene.export).  Host-only, numpy + the standard library.

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
FLOAT, UNSIGNED_BYTE, ARRAY_BUFFER, POINTS = 5126, 5121, 34962, 0


def _numpy(t) -> np.ndarray:
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


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
    node = {"mesh": 0}
    if cloud.get("align") is not None:
        m = np.asarray(_numpy(cloud["align"]), dtype=np.float64).reshape(4, 4)
        node["matrix"] = [float(v) for v in m.T.reshape(-1)]             # column-major
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
    js = json.dumps(doc, separators=(",", ":")).encode()
    js += b" " * (-len(js) % 4)                           # chunks are padded to 4 bytes: JSON with spaces, BIN with zeros
    binary += b"\0" * (-len(binary) % 4)
    total = 12 + 8 + len(js) + 8 + len(binary)
    return (struct.pack("<III", GLB_MAGIC, 2, total) + struct.pack("<II", len(js), CHUNK_JSON) + js
            + struct.pack("<II", len(binary), CHUNK_BIN) + binary)


def write_glb(path: str, cloud: dict) -> None:
    """Write ``cloud`` (``OmniVGGT.point_cloud`` output) to ``path`` as a glTF 2.0 binary file."""
    data = glb_bytes(cloud)
    with open(path, "wb") as f:
        f.write(data)
