"""Independence from the memory a call is handed (GPU): every buffer the package allocates with torch.empty / empty_like is
filled with a poison pattern and fenced by guard bands, and each entry point must return bit for bit what it returns on
ordinary memory, finite where it must be, inside its buffers, and still pass the reference check its own test applies.

The ``poisoned`` context replaces the ``torch`` name of the package modules with a proxy whose ``empty`` / ``empty_like``
allocate GUARD + n + GUARD bytes, fill the middle with the poison byte and both guard bands with GUARD_BYTE, and return the
middle.  torch.zeros is left alone (zeroed buffers are zero on purpose) but recorded.  Patterns: 0xFF (NaN in every float
type, -1 in signed integers), 0x00 (what fresh memory usually holds), and 0x3F on float tensors (0.747 in fp32: a finite
value that max and comparisons do not drop) with 0xFF on integer tensors, so an index or a count only ever starts as 0 or -1.
Between calls and graph replays the engine's Workspace.bufs and the static outputs of every captured graph are poisoned again.

Which launch first writes each stateful region, per entry point (read from csrc/):
  aggregator   has_depth / depth_rows: aux_index_kernel; the residual stream x: assemble_tokens_kernel (every token row);
               depth scratch (fp64 partial sums + scale): depth_stats_kernel writes every chunk's partials, depth_scale_kernel
               reads them; depth im2col rows: depth_im2col_kernel (every column, including the padding columns).
  DINOv2       x and the patch-row list: dino_init_kernel; image im2col rows: image_im2col_kernel (padding columns zeroed).
  attention    KV-split partials (part_o, part_ml): the split CTAs of the same launch, before attn_merge_kernel.
  DPT head     feat[l] zero borders: cudaMemsetAsync in ovg_dpt_forward (the DENSE2PAD / PIXSHUF stores write the interior only);
               lr, t, u, v, w, o1 borders: the ROWS_PAD epilogue writes border rows as zeros; xl[l] borders:
               upsample_rows_kernel / upsample_bilinear_kernel write rows 0 and H + 1 and the border columns as zeros;
               colsd: im2col3x3s2_kernel writes zeros for taps outside the map; tail scratch (gx, gy): tail_tables_kernel.
  camera head  pose: pose_out_kernel of iteration 0 (pose_embed_silu reads the empty pose token then, not the buffer).
  percentile   state, histograms and the kept counter: select_init_kernel; histograms re-zeroed by select_decide_kernel.
  point cloud  tile_count: cloud_count_kernel (every tile); tile_offset and the count: tile_scan_kernel; centre partials:
               cloud_center_partial_kernel (all CLOUD_CENTER_BLOCKS blocks).
  matches      flag, histograms, cell counts: cudaMemsetAsync in ovg_match_index; per-view counts and offsets: the keep count
               and scan kernels; the pair counts: ovg_match_query.
  sky          labels, areas and per-view maxima: the init kernel of ovg_segment_sky.
  FPS          grid arrival counters: cudaMemsetAsync in ovg_farthest_point_sample.
  ranking      histograms live in shared memory; keys and scales: the first of the two launches.
  Sim(3)       part0 (count and sums): every block of sim3_means_kernel; part1 (moments): every block of sim3_moments_kernel;
               part2 (squared residuals): every block of sim3_residual_kernel; the status word stats[1]: sim3_solve_kernel.
  JPEG         status words, exit and changed flags, and the whole 64-coefficient blocks: cudaMemsetAsync in ovg_jpeg_decode.
  loaders      resized views: resize_v_u8_f32_kernel writes every pixel of its output frame (the pad fill included);
               w2c / K: camera_prepare_kernel, zeros for a view without a camera; depth and mask maps are torch.zeros.
Context parallelism is not covered: its peer flags and epoch counter are persistent by design and it needs two GPUs."""
import contextlib
import functools
import importlib
import sys

import numpy as np
import pytest
import torch

from ovg_support import randn, scene

GUARD = 4096                 # keeps the 256-byte workspace and 16-byte TMA alignment of the allocator's blocks
GUARD_BYTE = 0x5A
PATTERNS = ("nan", "zero", "finite")
_BYTES = {"nan": (0xFF, 0xFF), "zero": (0x00, 0x00), "finite": (0x3F, 0xFF)}     # (float tensors, other tensors)
PACKAGE_MODULES = ("ops", "engine", "model", "scene", "geometry", "preprocess", "pipeline", "torch_parts")


def _kind(frame, shape, dtype) -> str:
    """'workspace' for the engine's named buffers (Workspace.get) and for flat integer buffers (every *_workspace_bytes /
    scratch allocation of the package is a 1-D uint8 tensor, the percentile's a 1-D int64 one), else 'output'.  Only the
    count of poisoned workspaces and the printed statistics depend on it."""
    if isinstance(frame.f_locals.get("self"), _engine().Workspace):
        return "workspace"
    return "workspace" if dtype in (torch.uint8, torch.int64) and len(shape) == 1 else "output"


def _engine():
    return importlib.import_module("omnivggt_official_b200.engine")


class PoisonTorch:
    """Stands in for the torch module inside the package: see the module docstring."""

    def __init__(self, pattern, devices=("cuda",)):
        self._pattern, self._devices = pattern, devices
        self.allocs = []        # (raw uint8 buffer, payload bytes, kind)
        self.zeroed = []        # tensors from torch.zeros on a poisoned device

    def __getattr__(self, name):
        return getattr(torch, name)

    def byte_for(self, dtype) -> int:
        return _BYTES[self._pattern][0 if dtype.is_floating_point else 1]

    def _device(self, device):
        return torch.device(device) if device is not None else torch.empty(0).device

    def empty(self, *size, dtype=None, device=None, **kw):
        shape = tuple(size[0]) if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else size
        dev = self._device(device)
        if dev.type not in self._devices or any(kw.values()):
            return torch.empty(*size, dtype=dtype, device=device, **kw)
        shape, dtype = tuple(int(s) for s in shape), dtype or torch.get_default_dtype()
        return self.alloc(shape, dtype, dev, _kind(sys._getframe(1), shape, dtype))

    def empty_like(self, t, *, dtype=None, device=None, **kw):
        dev = self._device(device if device is not None else t.device)
        if dev.type not in self._devices or any(kw.values()):
            return torch.empty_like(t, dtype=dtype, device=device, **kw)
        return self.alloc(tuple(t.shape), dtype or t.dtype, dev, _kind(sys._getframe(1), tuple(t.shape), dtype or t.dtype))

    def zeros(self, *a, **kw):
        t = torch.zeros(*a, **kw)
        if t.device.type in self._devices:
            self.zeroed.append(t)
        return t

    def alloc(self, shape, dtype, device, kind="output"):
        n = int(np.prod(shape, dtype=np.int64)) * torch.empty((), dtype=dtype).element_size()
        raw = torch.empty(2 * GUARD + n, dtype=torch.uint8, device=device)
        raw.fill_(GUARD_BYTE)
        mid = raw[GUARD:GUARD + n]
        mid.fill_(self.byte_for(dtype))
        self.allocs.append((raw, n, kind))
        return mid.view(dtype).view(shape)

    def refill(self, t):
        """Poison an existing contiguous tensor again (a persistent workspace or a graph's static output)."""
        if torch.is_tensor(t) and t.numel() and t.is_contiguous():
            t.view(-1).view(torch.uint8).fill_(self.byte_for(t.dtype))

    def repoison_model(self, m):
        if m._engine is not None:
            for t in m._engine.ws.bufs.values():
                self.refill(t)
        for ent in m._graphs.values():
            for k, v in ent.get("out", {}).items():
                if k != "images":
                    for t in (v if isinstance(v, list) else [v]):
                        self.refill(t)

    def guards_broken(self):
        """Allocations whose guard bands changed (one device read for all of them)."""
        if not self.allocs:
            return []
        bad = torch.stack([((raw[:GUARD] != GUARD_BYTE).any() | (raw[GUARD + n:] != GUARD_BYTE).any())
                           for raw, n, _ in self.allocs]).cpu()
        return [i for i, b in enumerate(bad.tolist()) if b]

    def ranges(self):
        """(start, end) device addresses of every payload the proxy handed out, zeroed buffers included."""
        out = [(raw.data_ptr() + GUARD, raw.data_ptr() + GUARD + n) for raw, n, _ in self.allocs]
        return out + [(t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()) for t in self.zeroed]

    def stats(self):
        ws = [n for _, n, k in self.allocs if k == "workspace"]
        return len(self.allocs), len(ws), sum(n for _, n, _ in self.allocs)


class _Unpoisoned:
    """The baseline run: same interface, ordinary memory."""

    def repoison_model(self, m):
        pass

    def refill(self, t):
        pass


@contextlib.contextmanager
def poisoned(pattern, devices=("cuda",)):
    mods = [importlib.import_module(f"omnivggt_official_b200.{n}") for n in PACKAGE_MODULES]
    proxy = PoisonTorch(pattern, devices)
    saved = [(m, m.torch) for m in mods]
    for m in mods:
        m.torch = proxy
    try:
        yield proxy
    finally:
        for m, t in saved:
            m.torch = t


@pytest.fixture()
def poison():
    """The context manager ``poisoned(pattern, devices)``."""
    return poisoned


# ------------------------------------------------------------------------------------------------------------------ harness
def _flat(obj, path=""):
    if torch.is_tensor(obj):
        return [(path, obj.detach().clone())]
    if isinstance(obj, dict):
        return [x for k in sorted(obj, key=str) for x in _flat(obj[k], f"{path}.{k}")]
    if isinstance(obj, (list, tuple)):
        return [x for i, v in enumerate(obj) for x in _flat(v, f"{path}[{i}]")]
    return [(path, obj)]


def _bits_equal(a, b):
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.numel() == 0:
        return True
    return torch.equal(a.contiguous().view(-1).view(torch.uint8), b.contiguous().view(-1).view(torch.uint8))


def check_case(name, run, finite=(), reference=None, need_workspace=True):
    """run(P) -> nested outputs; P is the poisoning proxy or the unpoisoned stand-in.  Asserts (a) bit equality with the
    unpoisoned run, (b) finiteness of every output whose path contains one of ``finite``, (c) intact guard bands and at least
    one poisoned workspace (a bare kernel call without one poisons its output), (d) ``reference(outputs)``."""
    want = _flat(run(_Unpoisoned()))
    torch.cuda.synchronize()
    for pattern in PATTERNS:
        with poisoned(pattern) as P:
            res = run(P)
            torch.cuda.synchronize()
        got = _flat(res)
        n_alloc, n_ws, nbytes = P.stats()
        broken = P.guards_broken()
        assert not broken, (name, pattern, [(P.allocs[i][1], P.allocs[i][2]) for i in broken])
        assert n_ws >= 1 or (not need_workspace and n_alloc >= 1), (name, pattern, "no workspace was poisoned")
        assert [p for p, _ in got] == [p for p, _ in want], (name, pattern)
        for (path, g), (_, w) in zip(got, want):
            if torch.is_tensor(w):
                assert _bits_equal(g, w), (name, pattern, path)
                if any(f in path for f in finite) and g.is_floating_point():
                    assert torch.isfinite(g).all(), (name, pattern, path)
            else:
                assert g == w, (name, pattern, path)
        if reference is not None:
            reference(res)
        print(f"{name} [{pattern}]: {n_alloc} allocations poisoned ({n_ws} workspaces), {nbytes} bytes, guards held")
        del P, res, got
        torch.cuda.empty_cache()


pytestmark = pytest.mark.gpu
DENSE = ("depth", "world_points", "pose_enc")


# ------------------------------------------------------------------------------------------------------------------ forward
def _golden():
    from conftest import golden_index
    return golden_index()


def _forward_calls(m, inp, kw, graphed, P):
    """One eager call, or four calls with CUDA graphs (two eager, a capture, a replay), everything re-poisoned in between."""
    m._invalidate()
    m.use_cuda_graph = graphed
    outs = []
    for i in range(4 if graphed else 1):
        if i:
            P.repoison_model(m)
        outs.append(m(**inp, **kw))
    if graphed:
        assert all(e["graph"] is not None for e in m._graphs.values())
    return outs


_MINI = {}


def _mini(variant):
    from test_model_gpu import build
    if variant not in _MINI:
        _MINI[variant] = build(variant)
    return _MINI[variant]


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("case", sorted(_golden()))
def test_forward_reduced(case, graphed):
    from oracle.synth import make_inputs
    from test_model_gpu import reduced_golden_check
    meta = _golden()[case]
    m = _mini(meta["variant"])
    inp = {k: v.cuda() for k, v in make_inputs(meta["B"], meta["S"], meta["H"], meta["W"], seed=meta["input_seed"]).items()}
    kw = dict(depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"])

    def reference(outs):
        for o in outs:
            reduced_golden_check(case, o)
    try:
        check_case(f"forward {case} {'graphs' if graphed else 'eager'}", lambda P: _forward_calls(m, inp, kw, graphed, P),
                   finite=DENSE, reference=reference)
    finally:
        m.use_cuda_graph, m._graphs = False, {}


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("case", ["full_cfg1", "full_tall_s3"])
def test_forward_full_size(case, graphed):
    from oracle.synth import make_inputs
    from test_model_gpu import FULL_INDEX, full_model, full_size_check, set_heads
    meta = FULL_INDEX[case]
    m = full_model()
    set_heads(m, "fp16")
    use = m.use_cuda_graph
    inp = {k: v.cuda() for k, v in make_inputs(1, meta["S"], meta["H"], meta["W"], seed=meta["input_seed"]).items()}
    kw = dict(depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"])

    def reference(outs):
        for i, o in enumerate(outs):
            full_size_check(case, o, f"heads=fp16 poisoned, call {i + 1}", log=False)
    try:
        check_case(f"forward {case} {'graphs' if graphed else 'eager'}", lambda P: _forward_calls(m, inp, kw, graphed, P),
                   finite=DENSE, reference=reference)
    finally:
        m.use_cuda_graph, m._graphs = use, {}
        m._invalidate()


def test_forward_full_size_smaller_call_gets_a_poisoned_prefix():
    """4 views of 518 x 518, then 3 views of 518 x 518 with depth and camera aux (every workspace of the second call is a
    prefix of the first call's, poisoned again: none is reallocated), then the 4 views again."""
    from oracle.synth import make_inputs
    from test_model_gpu import FULL_INDEX, full_model, full_size_check, set_heads
    m = full_model()
    set_heads(m, "fp16")
    use = m.use_cuda_graph
    seq = ["full_cfg1", "full_aux_s3", "full_cfg1"]
    inputs = {}
    for case in set(seq):
        meta = FULL_INDEX[case]
        inputs[case] = ({k: v.cuda() for k, v in make_inputs(1, meta["S"], meta["H"], meta["W"], seed=meta["input_seed"]).items()},
                        dict(depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"]))

    def run(P):
        m._invalidate()
        m.use_cuda_graph = False
        outs = []
        for i, case in enumerate(seq):
            if i:
                P.repoison_model(m)
            version = m._engine.ws.version if i else None
            outs.append(m(**inputs[case][0], **inputs[case][1]))
            assert version is None or m._engine.ws.version == version, "a workspace was reallocated"
        return outs

    def reference(outs):
        for case, o in zip(seq, outs):
            full_size_check(case, o, "heads=fp16 poisoned, size sequence", log=False)
        for k in DENSE:
            assert torch.equal(outs[0][k], outs[2][k]), k
    try:
        check_case("forward 518 S=4, S=3 with aux, S=4", run, finite=DENSE, reference=reference)
    finally:
        m.use_cuda_graph, m._graphs = use, {}
        m._invalidate()


# ------------------------------------------------------------------------------------------------------------------ components
def test_components():
    """model.aggregator (fp32 layer export), camera_head, depth_head and point_head on those layers, against the reduced
    golden of the same inputs."""
    from oracle.synth import make_inputs
    from test_model_gpu import reduced_golden_check
    case = "conv_partial_aux_b2"
    meta = _golden()[case]
    m = _mini(meta["variant"])
    inp = {k: v.cuda() for k, v in make_inputs(meta["B"], meta["S"], meta["H"], meta["W"], seed=meta["input_seed"]).items()}

    def run(P):
        m._invalidate()
        layers, psi = m.aggregator(**inp, depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"])
        P.repoison_model(m)
        cams = m.camera_head(layers)
        P.repoison_model(m)
        depth, dconf = m.depth_head(layers, inp["images"], psi)
        P.repoison_model(m)
        pts, pconf = m.point_head(layers, inp["images"], psi, frames_chunk_size=1)
        return {"layers": layers, "pose_enc": cams[-1], "pose_enc_list": cams, "depth": depth, "depth_conf": dconf,
                "world_points": pts, "world_points_conf": pconf}

    check_case("components", run, finite=DENSE + ("layers",), reference=lambda o: reduced_golden_check(case, o))


@pytest.mark.parametrize("drop", [("depth_head",), ("point_head",), ("depth_head", "point_head")])
def test_forward_without_dpt_heads(drop):
    from oracle.synth import make_inputs
    from test_model_gpu import build, reduced_golden_check
    case = "conv_full_aux_rect"
    meta = _golden()[case]
    m = build(meta["variant"])
    for name in drop:
        setattr(m, name, None)
    inp = {k: v.cuda() for k, v in make_inputs(meta["B"], meta["S"], meta["H"], meta["W"], seed=meta["input_seed"]).items()}
    kw = dict(depth_gt_index=meta["depth_gt_index"], camera_gt_index=meta["camera_gt_index"])
    keys = ["pose_enc"] + [k for h, ks in (("depth_head", ("depth", "depth_conf")), ("point_head", ("world_points", "world_points_conf")))
                           if h not in drop for k in ks]

    def reference(outs):
        for o in outs:
            reduced_golden_check(case, o, keys)
    for graphed in (False, True):
        check_case(f"forward without {drop} {graphed}", lambda P: _forward_calls(m, inp, kw, graphed, P), finite=DENSE,
                   reference=reference)


# ------------------------------------------------------------------------------------------------------------------ post-processing
_PRED = {}


def _predictions():
    """One unpoisoned forward of the mini model (3 views of 56 x 56): the input of the post-processing cases."""
    if "p" not in _PRED:
        from oracle.synth import make_inputs
        m = _mini("mini_conv")
        inp = {k: v.cuda() for k, v in make_inputs(1, 3, 56, 56, seed=4).items()}
        _PRED["p"] = {k: v for k, v in m(depth_gt_index=[1], camera_gt_index=[0], **inp).items()}
    return _PRED["p"]


def test_postprocess():
    from test_postprocess import check_postprocess_against_oracle
    raw = _predictions()
    m = _mini("mini_conv")
    # (the mini model's random field-of-view outputs can give infinite focal lengths, so intrinsics and the unprojected points
    # are held to bit equality and the oracle, not to finiteness)
    check_case("postprocess", lambda P: {k: v for k, v in m.postprocess(dict(raw), conf_percent=25.0).items() if k not in raw},
               finite=("extrinsic", "conf_threshold"), reference=lambda o: check_postprocess_against_oracle({**raw, **o}, 25.0))


def test_conf_percentile_mask_odd_length():
    from omnivggt_official_b200 import ops
    g = torch.Generator().manual_seed(3)
    conf = 1.0 + torch.rand(7 * 1001 + 3, generator=g).pow(3) * 8.0
    conf[::5] = conf[0]
    c = conf.cuda()

    def reference(o):
        mask, thr, cnt = o
        t = np.percentile(conf.numpy(), 42.0)
        assert float(thr) == float(t), (float(thr), t)
        want = (c >= thr) & (c > 0.1)
        assert torch.equal(mask.bool(), want) and int(cnt) == int(want.sum())
    check_case("conf_percentile_mask", lambda P: ops.conf_percentile_mask(c, 42.0, 0.1), finite=("",), reference=reference)


@pytest.mark.parametrize("kind", ["glb", "viewer"])
def test_point_cloud_filter_modes(kind):
    from oracle.make_golden_cloud import GLB_CASES, VIEWER_CASES
    from test_point_cloud import _check_against_oracle, _device_cloud, _gold, _source
    g = _gold()
    if kind == "glb":
        src, pct, frame, black, white = GLB_CASES[1]
        world, conf = _source(g, src)
        floor, kw = 1e-5, dict(conf_percent=pct, frame=frame, mask_black_bg=black, mask_white_bg=white)
    else:
        pct, black, white = VIEWER_CASES[0]
        world, conf, frame = g["world_points_from_depth"], g["depth_conf"], None
        floor, kw = 0.1, dict(conf_percent=pct, conf_floor=0.1, mask_black_bg=black, mask_white_bg=white)

    def run(P):
        return {k: torch.from_numpy(v) for k, v in _device_cloud(world, conf, g["images"], g["extrinsic"], **kw).items()}

    def reference(o):
        _check_against_oracle({k: v.numpy() for k, v in o.items()}, world, conf, g["images"], g["extrinsic"], pct, floor, frame,
                              black, white)
    check_case(f"point_cloud {kind}", run, finite=("points", "center", "scale", "align"), reference=reference)


def _scene_cuda(S=3, H=40, W=48, seed=3):
    return {k: v.cuda() for k, v in scene(S, H, W, seed, distinct_cameras=True).items()}


def _host_sky(images):
    """The sky oracle on every view of images fp32 [S, 3, H, W]: bool [S, H, W]."""
    from oracle import sky_oracle as SKO
    h = images.cpu().numpy()
    return np.stack([SKO.segment_sky(np.ascontiguousarray(v.transpose(1, 2, 0))) for v in h])


def test_point_cloud_mask_sky():
    """mask_sky=True against the cloud built with the sky oracle's masks."""
    from omnivggt_official_b200 import OmniVGGT
    from test_sky import _blob_images
    pred = _scene_cuda()
    pred["images"] = _blob_images(3, 40, 48, seed=1)[None].cuda()
    sky = _host_sky(pred["images"][0])
    assert sky.any() and not sky.all()

    def reference(o):
        want = OmniVGGT.point_cloud(pred, mask_sky=torch.from_numpy(sky).cuda())
        assert len(o["points"]) > 0
        for k in want:
            assert torch.equal(o[k], want[k]), k
    check_case("point_cloud mask_sky", lambda P: OmniVGGT.point_cloud(pred, mask_sky=True), finite=("points", "center", "scale"),
               reference=reference)


def test_point_cloud_max_points():
    """max_points: the reference's farthest_point_sample over the full cloud's points."""
    from omnivggt_official_b200 import OmniVGGT
    from oracle import fps_oracle as FO
    pred = _scene_cuda()
    full = OmniVGGT.point_cloud(pred, mask_black_bg=True)
    assert len(full["points"]) > 500
    idx = torch.from_numpy(FO.farthest_point_sample(full["points"][None].cpu().numpy(), 500)[0]).cuda()

    def reference(o):
        for k in ("points", "colors", "frame"):
            assert torch.equal(o[k], full[k][idx]), k
    check_case("point_cloud max_points", lambda P: OmniVGGT.point_cloud(pred, max_points=500, mask_black_bg=True),
               finite=("points", "center", "scale"), reference=reference)


@pytest.mark.parametrize("layout", ["reference", "glb"])
def test_mesh(layout):
    from omnivggt_official_b200 import OmniVGGT
    from oracle.make_golden_cloud import GLB_CASES
    from test_mesh import _check_device_against_oracle, _np, _pred, _source
    from test_point_cloud import _gold
    g = _gold()
    src, pct, frame, black, white = GLB_CASES[1]
    world, conf = _source(g, src)
    pred = _pred(g)

    def reference(o):
        d = _np(o)
        assert len(d["faces" if layout == "reference" else "indices"]) > 0
        _check_device_against_oracle(d, world, conf, g["images"], g["extrinsic"], pct, frame, black, white, layout)
    check_case(f"mesh {layout}", lambda P: OmniVGGT.mesh(pred, source=src, conf_percent=pct, frame=frame, mask_black_bg=black,
                                                         mask_white_bg=white, layout=layout), reference=reference)


def test_matches():
    from omnivggt_official_b200 import OmniVGGT, ops
    from oracle import matches_oracle as MO
    from test_matches import _scene
    pred = {k: v.cuda() for k, v in _scene(3, 40, 48).items()}

    def reference(o):
        mask, _, _ = ops.conf_percentile_mask(pred["depth_conf"][0].contiguous(), 20.0, 1e-5)
        ref = MO.scene_matches(pred["world_points_from_depth"][0].cpu().numpy(), mask.bool().cpu().numpy(), [(0, 1), (0, 2), (1, 2)])
        assert len(o) == 3 and all(r["count"] > 0 for r in ref)
        for a, r in zip(o, ref):
            assert a["count"] == r["count"]
            assert np.array_equal(a["xy_i"].cpu().numpy(), r["xy_i"]) and np.array_equal(a["xy_j"].cpu().numpy(), r["xy_j"])
    check_case("matches", lambda P: OmniVGGT.matches(pred, conf_percent=20.0), reference=reference)


def test_sky_mask():
    from omnivggt_official_b200 import OmniVGGT
    from test_sky import _blob_images
    images = _blob_images(3, 64, 80, seed=2).cuda()
    want = _host_sky(images)
    assert want.any() and not want.all()
    check_case("sky_mask", lambda P: OmniVGGT.sky_mask({"images": images[None]}),
               reference=lambda o: np.array_equal(o.cpu().numpy(), want) or pytest.fail("sky differs from the oracle"))


# ------------------------------------------------------------------------------------------------------------------ geometry
@pytest.mark.parametrize("size", ["cta_b3_odd", "grid_above_threshold", "grid_streamed_surface_8x518"])
def test_farthest_point_sample(size):
    from omnivggt_official_b200 import ops
    from oracle import fps_oracle as FO
    from test_fps import SIZES
    make, npoint, ends = SIZES[size]
    xyz = make().cuda().contiguous()
    start = torch.randint(0, xyz.shape[1], (xyz.shape[0],), generator=torch.Generator().manual_seed(9)).cuda()
    want = FO.farthest_point_sample_torch(xyz, npoint, ends, start)
    check_case(f"fps {size}", lambda P: ops.farthest_point_sample(xyz, npoint, start, ends),
               reference=lambda o: torch.equal(o, want) or pytest.fail("fps differs from the restatement"))


@pytest.mark.parametrize("N,batched", [(8192, False), (6001, True), (8193, True)], ids=["smem_f64", "smem_f32", "grid"])
def test_compute_ranking(N, batched):
    from omnivggt_official_b200.geometry import compute_ranking
    from test_ranking import _large, _self_consistent
    E = torch.from_numpy(_large(N, seed=N)).cuda()

    def reference(o):
        ranking, dists = o
        assert dists.dtype == (torch.float64 if not batched or N <= 6000 else torch.float32)
        assert _self_consistent(ranking, dists)
    check_case(f"compute_ranking {N}", lambda P: compute_ranking(E, batched=batched), finite=("",), reference=reference)


def test_find_reciprocal_matches():
    from omnivggt_official_b200.geometry import find_reciprocal_matches
    from oracle import matches_oracle as MO
    from oracle.make_golden_matches import surface_views
    sv = surface_views(S=2, H=40, W=48, seed=3).reshape(2, -1, 3)
    P1, P2 = sv[0][::2].copy(), sv[1][1::3].copy()
    want = MO.find_reciprocal_matches(P1, P2)

    def reference(o):
        rec, nn, count = o
        assert np.array_equal(rec.cpu().numpy(), want[0]) and np.array_equal(nn.cpu().numpy(), want[1]) and count == want[2]
    check_case("find_reciprocal_matches", lambda P: find_reciprocal_matches(torch.from_numpy(P1).cuda(), torch.from_numpy(P2).cuda()),
               reference=reference)


@pytest.mark.parametrize("name", ["noise", "outliers_masked", "n65537"])
def test_align_sim3(name):
    from omnivggt_official_b200 import geometry
    from oracle import sim3_oracle as SO
    from test_long_capture import CASES, _rel
    src, dst, keep = CASES[name]
    ref, _ = SO.umeyama(src, dst, keep)
    check_case(f"align_sim3 {name}", lambda P: geometry.align_sim3(src, dst, keep), finite=("",),
               reference=lambda o: _rel(o.cpu().numpy(), ref) < 1e-9 or pytest.fail("sim3 differs from the oracle"))


@pytest.mark.parametrize("overlap", [1, 3])
def test_reconstruct(overlap):
    from oracle.synth import make_inputs
    m = _mini("mini_conv")
    inp = {k: v.cuda() for k, v in make_inputs(1, 13, 56, 56, seed=63).items()}

    def run(P):
        m._invalidate()
        return m.reconstruct(**inp, chunk=8, overlap=overlap)

    def reference(o):
        """The schedule, a positive alignment count at every set boundary, and the first set equal to the plain forward
        (test_long_capture checks the later sets against the Sim(3) oracle)."""
        from oracle import sim3_oracle as SO
        assert o["chunks"] == SO.schedule(13, 8, overlap) and len(o["chunks"]) > 1
        assert (o["align_pairs"][1:] > 0).all() and (o["align_pairs"][:1] == 0).all()
        raw = m(**{k: v[:, :8] for k, v in inp.items()})
        assert torch.equal(o["depth"][0, :8], raw["depth"][0]) and torch.equal(o["depth_conf"][0, :8], raw["depth_conf"][0])
    check_case(f"reconstruct overlap {overlap}", run, finite=("depth", "world_points", "extrinsic", "sim3"), reference=reference)


# ------------------------------------------------------------------------------------------------------------------ input pipeline
def test_decode_images(tmp_path):
    from test_jpeg import _device_decode, corrupted, matrix, pillow_rgb
    files = [f for f in matrix() if f[0].split("-")[1] in ("s420", "rst3") or f[0].startswith(("3x5", "17x33"))]
    files.append(("flagged", corrupted()[0]))

    def reference(outs):
        for (name, data), t in zip(files, outs):
            assert np.array_equal(t.cpu().numpy(), pillow_rgb(data)), name
    check_case("decode_images", lambda P: _device_decode(tmp_path, files), reference=reference)


@pytest.mark.parametrize("mode", ["crop", "pad"])
def test_load_and_preprocess_images(mode, tmp_path):
    from omnivggt_official_b200 import preprocess as PP
    from oracle import jpeg_oracle as J
    from test_jpeg import _write
    files = [(f"v{i}", J.encode(J.octave_noise(w, h, seed=i))) for i, (w, h) in enumerate([(640, 480), (300, 500), (97, 61)])]
    paths = sorted(_write(str(tmp_path), files))
    want = PP.preprocess_images([PP.decode_rgb(p) for p in paths], mode)          # host (Pillow) decode, same device resize

    check_case(f"load_and_preprocess_images {mode}", lambda P: PP.load_and_preprocess_images(paths, mode=mode), finite=("",),
               reference=lambda o: torch.equal(o, want) or pytest.fail("differs from the host-decoded images"))


@pytest.mark.parametrize("name", ["wide", "tall"])
def test_load_images_and_cameras(name, tmp_path):
    """A synthetic folder with .npy and transposed 16-bit .png depth maps and one view without a camera file (its w2c and K
    are the zeros camera_prepare_kernel writes), against the oracle loader and the reference loader's digests.  The views are
    PNG, decoded on the host: the poisoned buffers are the loader's outputs and its resize temporaries."""
    from omnivggt_official_b200 import preprocess as PP
    from oracle.synth_folder import make_folder
    from test_preprocess import check_pipeline_against_oracle
    d = make_folder(str(tmp_path), name, seed=0)
    check_case(f"load_images_and_cameras {name}", lambda P: PP.load_images_and_cameras(d["images"], d["cameras"], d["depths"]),
               finite=("[0]", "[1]", "[2]", "[3]", "[4]"), reference=lambda o: check_pipeline_against_oracle(name, d, o),
               need_workspace=False)


# ------------------------------------------------------------------------------------------------------------------ kernel entry points
_randn = functools.partial(randn, host_rng=True)


def _to_pad(x, dtype):
    return torch.nn.functional.pad(x.permute(0, 2, 3, 1), (0, 0, 1, 1, 1, 1)).to(dtype).contiguous()


def test_dpt_tail_scratch():
    from omnivggt_official_b200 import ops
    Fr, h, w, H, W, Cin = 2, 12, 20, 21, 35, 128
    xp = _to_pad(_randn(Fr, Cin, h, w, seed=1), torch.float16)
    wb = _randn(32, 9 * Cin, scale=(9 * Cin) ** -0.5, seed=2).to(torch.float16)
    b1, w2, b2 = _randn(32, scale=0.1, seed=3), _randn(4, 32, scale=32 ** -0.5, seed=4), _randn(4, scale=0.1, seed=5)
    tx, ty = _randn(W, Cin // 2, scale=0.1, seed=6), _randn(H, Cin // 2, scale=0.1, seed=7)
    check_case("dpt_tail", lambda P: ops.dpt_tail(xp, tx, ty, wb, b1, w2, b2, 1, Fr, h, w, H, W), finite=("",))


def _alloc(P, shape, dtype, kind="output"):
    """A test-owned buffer: poisoned under the proxy, zeros in the unpoisoned run."""
    if isinstance(P, PoisonTorch):
        return P.alloc(shape, dtype, torch.device("cuda"), kind)
    return torch.zeros(shape, dtype=dtype, device="cuda")


def test_depth_im2col_scratch():
    from omnivggt_official_b200 import ops
    B, S, H, W, patch = 2, 4, 28, 42, 14
    idx = torch.tensor([0, 2, 3], device="cuda", dtype=torch.int32)
    g = torch.Generator().manual_seed(0)
    depth = (0.5 + 4 * torch.rand(B, S, H, W, generator=g)).cuda()
    mask = (torch.rand(B, S, H, W, generator=g) > 0.3).float().cuda()
    mask[1] = 0
    Sd, P_ = 3, (H // patch) * (W // patch)

    def run(P):
        cols = _alloc(P, (B * Sd * P_, 2 * patch * patch), torch.bfloat16)
        scratch = _alloc(P, (ops.L.DEPTH_SCRATCH_DOUBLES(B),), torch.float64, "workspace")
        ops.depth_im2col(depth, mask, idx, scratch, cols, B, S, Sd, H, W, patch)
        return cols
    check_case("depth_im2col", run, finite=("",))


@pytest.mark.parametrize("rowmap", ["HEADTAIL", "PIXSHUF", "DENSE2PAD", "PAD"])
def test_gemm_row_maps(rowmap):
    """GEMM stores into poisoned outputs: the PAD rows map writes its border rows as zeros; PIXSHUF and DENSE2PAD write the
    interior only and leave the border (which their callers zero) as it was."""
    from omnivggt_official_b200 import ops
    L, BF = ops.L, torch.bfloat16
    Fr, h, w, C = 2, 9, 7, 64
    bias = _randn(C, seed=3)
    taps = [(ky - 1) * (w + 2) + (kx - 1) for ky in range(3) for kx in range(3)]

    def run(P):
        if rowmap == "HEADTAIL":
            xp = _to_pad(_randn(Fr, 128, h, w, seed=1), BF)
            wb = _randn(32, 9 * 128, scale=(9 * 128) ** -0.5, seed=2).to(BF)
            preds, conf = _alloc(P, (Fr, h, w, 3), torch.float32), _alloc(P, (Fr, h, w), torch.float32)
            ops.gemm(xp.reshape(-1, 128), wb, taps=taps, epi=L.EPI_HEADTAIL, bias=_randn(32, seed=3), w2=_randn(4, 32, seed=4),
                     b2=_randn(4, seed=5), outc=4, head_act=1, preds=preds, conf=conf, rowmap=L.ROWS_PAD, gh=h, gw=w)
            return preds, conf
        if rowmap == "PAD":
            xp = _to_pad(_randn(Fr, C, h, w, seed=1), BF)
            out = _alloc(P, (Fr, h + 2, w + 2, C), BF)
            ops.gemm(xp.reshape(-1, C), _randn(C, 9 * C, scale=(9 * C) ** -0.5, seed=2).to(BF), taps=taps, epi=L.EPI_BF16,
                     bias=bias, act=L.ACT_RELU, out=out, ldo=C, rowmap=L.ROWS_PAD, gh=h, gw=w)
            border = out.clone()
            border[:, 1:-1, 1:-1] = 0
            assert (border == 0).all(), "the PAD row map must write its border rows as zeros"
            return out
        ps = 2 if rowmap == "PIXSHUF" else 1
        out = _alloc(P, (Fr, h * ps + 2, w * ps + 2, C), BF)
        a = _randn(Fr * h * w, C, seed=1).to(BF)
        if rowmap == "PIXSHUF":
            ops.gemm(a, _randn(ps * ps * C, C, scale=C ** -0.5, seed=2).to(BF), epi=L.EPI_BF16, bias=bias, out=out, ldo=C,
                     rowmap=L.ROWS_PIXSHUF, gh=h, gw=w, ps=ps, cout=C)
        else:
            ops.gemm(a, _randn(C, C, scale=C ** -0.5, seed=2).to(BF), epi=L.EPI_BF16, bias=bias, table=_randn(h * w, C, seed=4),
                     table_rows=h * w, out=out, ldo=C, rowmap=L.ROWS_DENSE2PAD, gh=h, gw=w)
        if isinstance(P, PoisonTorch):
            b = P.byte_for(BF)
            pv = (b << 8 | b) - (65536 if b >= 0x80 else 0)          # the poison as int16
            v = out.view(torch.int16)
            for edge in (v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1]):
                assert (edge == pv).all(), "the border rows must be left as they were"
        return out[:, 1:-1, 1:-1].contiguous()
    check_case(f"gemm {rowmap}", run, finite=("",), need_workspace=False)
