"""Sample layout and comparison of the full-size reference fixtures (tests/golden/full_*.safetensors)  --  TEST INFRASTRUCTURE.

A fixture keeps the reference's dense outputs (depth, depth_conf, world_points, world_points_conf at 518 x 518) only at a row
list x column list, and the pose encodings whole.  Each list is every ``stride``-th line from ``offset`` plus the BORDER outermost
lines at both ends, so the zero-bordered feature maps, the last tail strip and the edge clamps of the resizes are compared too.
The lists are stored per case in full_index.json ("rows", "cols"); tests read them from there and never rebuild them.

``compare`` turns a model output and a fixture into metrics: rel-L2 per output over all samples, per view, per border line,
per ``pose_enc_list`` entry, and the max-abs ``pose_enc`` error per view.  ``check`` asserts them against bars and names the view,
line or output that is over.  One number per output would hide a bad view: at 24 views, one view 3 % off everywhere moves the
aggregate by only ~0.03 / sqrt(24) = 6e-3.
"""
from __future__ import annotations

import json
import os
from typing import Dict, List

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
DENSE = ("depth", "depth_conf", "world_points", "world_points_conf")
BORDER = 2          # outermost lines per side that every fixture samples
PATCH = 14

# Bars at full size (DESIGN.md §2).  pose_enc_list entries are held to the aggregate bar.
BARS = dict(aggregate=1e-2, view=1.5e-2, border=1.5e-2, pose_enc_maxabs=5e-2)


def lines(n: int, stride: int, offset: int) -> List[int]:
    """Sample lines of an n-pixel axis: every stride-th from offset, plus the BORDER outermost lines at each end."""
    return sorted(set(range(offset, n, stride)) | set(range(BORDER)) | set(range(n - BORDER, n)))


def index() -> Dict[str, dict]:
    with open(os.path.join(GOLDEN, "full_index.json")) as f:
        return json.load(f)


def load(case: str) -> Dict[str, torch.Tensor]:
    from safetensors.torch import load_file
    return load_file(os.path.join(GOLDEN, f"{case}.safetensors"))


def sample(out: dict, rows: List[int], cols: List[int]) -> Dict[str, torch.Tensor]:
    """Model outputs (dense maps [B, S, H, W, ...]) -> what a fixture stores: the dense maps at rows x cols, pose_enc and each
    pose_enc_list entry, all fp32 on the host and owning their memory (pose_enc is the last list entry)."""
    store = {"pose_enc": out["pose_enc"].detach().float().cpu().clone()}
    for i, p in enumerate(out["pose_enc_list"]):
        store[f"pose_enc_list.{i}"] = p.detach().float().cpu().clone()
    for k in DENSE:
        t = out[k].detach()
        r = torch.as_tensor(rows, device=t.device)
        c = torch.as_tensor(cols, device=t.device)
        store[k] = t.index_select(2, r).index_select(3, c).float().cpu().clone()
    return store


def _rel(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def compare(got: Dict[str, torch.Tensor], ref: Dict[str, torch.Tensor], meta: dict) -> dict:
    """Metrics of a sampled output ``got`` (see ``sample``) against the fixture ``ref`` of the case described by ``meta``.

    aggregate[k]       rel-L2 over all samples of output k (dense outputs, pose_enc, pose_enc_list.i)
    view[k][s]         rel-L2 of dense output k over view s
    border[k][line]    rel-L2 of dense output k over one border line ("row 0", "col 517", ...), all views
    pose_enc_maxabs[s] max |pose_enc - ref| of view s
    """
    H, W = meta["H"], meta["W"]
    rows, cols = meta["rows"], meta["cols"]
    m = {"aggregate": {}, "view": {}, "border": {}}
    for k in ref:
        assert got[k].shape == ref[k].shape, (k, tuple(got[k].shape), tuple(ref[k].shape))
        m["aggregate"][k] = _rel(got[k], ref[k])
    edge = set(range(BORDER)) | set(range(H - BORDER, H))
    for k in DENSE:
        g, r = got[k], ref[k]
        m["view"][k] = [_rel(g[:, s], r[:, s]) for s in range(r.shape[1])]
        b = {}
        for i, y in enumerate(rows):
            if y in edge:
                b[f"row {y}"] = _rel(g[:, :, i], r[:, :, i])
        edge_w = set(range(BORDER)) | set(range(W - BORDER, W))
        for j, x in enumerate(cols):
            if x in edge_w:
                b[f"col {x}"] = _rel(g[:, :, :, j], r[:, :, :, j])
        m["border"][k] = b
    d = (got["pose_enc"].double() - ref["pose_enc"].double()).abs()
    m["pose_enc_maxabs"] = [d[:, s].max().item() for s in range(d.shape[1])]
    return m


def worst(metrics: dict) -> dict:
    """The largest value of each metric per output, with the view or line it is at, to 4 digits (for logs and DESIGN.md)."""
    def top(pairs):
        at, v = max(pairs, key=lambda t: t[1])
        return [at, float(f"{v:.4g}")]
    return {"aggregate": {k: float(f"{v:.4g}") for k, v in metrics["aggregate"].items()},
            "view": {k: top(enumerate(v)) for k, v in metrics["view"].items()},
            "border": {k: top(v.items()) for k, v in metrics["border"].items()},
            "pose_enc_maxabs": top(enumerate(metrics["pose_enc_maxabs"]))}


def check(metrics: dict, bars: dict = BARS) -> None:
    """Assert every metric is under its bar; the message names each failing output with its worst view or border line."""
    bad = []
    for k, v in metrics["aggregate"].items():
        if not v < bars["aggregate"]:
            bad.append(f"{k}: aggregate rel-L2 {v:.3g} >= {bars['aggregate']:.3g}")
    for k, per in metrics["view"].items():
        over = [s for s, v in enumerate(per) if not v < bars["view"]]
        if over:
            s = max(over, key=lambda i: per[i])
            bad.append(f"{k}: view {s} rel-L2 {per[s]:.3g} >= {bars['view']:.3g} (views over the bar: {over})")
    for k, per in metrics["border"].items():
        over = [n for n, v in per.items() if not v < bars["border"]]
        if over:
            n = max(over, key=lambda i: per[i])
            bad.append(f"{k}: border {n} rel-L2 {per[n]:.3g} >= {bars['border']:.3g} (lines over the bar: {over})")
    per = metrics["pose_enc_maxabs"]
    over = [s for s, v in enumerate(per) if not v < bars["pose_enc_maxabs"]]
    if over:
        s = max(over, key=lambda i: per[i])
        bad.append(f"pose_enc: view {s} max-abs {per[s]:.3g} >= {bars['pose_enc_maxabs']:.3g} (views over the bar: {over})")
    assert not bad, "; ".join(bad)
