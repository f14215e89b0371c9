"""Drop-in ``OmniVGGT`` module: the reference's constructor / forward / state-dict contract
(reference omnivggt/models/omnivggt.py:10-68, consumed by inference.py:321-356) on the H100-native engine.

    model = OmniVGGT().to("cuda").eval()
    model.load_state_dict(load_file("checkpoints/OmniVGGT.safetensors"))     # strict, same 1 505 keys
    predictions = model(images=..., extrinsics=..., intrinsics=..., depth=..., mask=...,
                        depth_gt_index=[...], camera_gt_index=[...])

Differences from the reference are additive only: aux tensors / index lists may be None, no network access at
construction, and extra keyword arguments select reduced architectures for tests.
"""
from __future__ import annotations

import os
import warnings
import weakref
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

try:  # keep from_pretrained / save_pretrained like the reference (omnivggt.py:3,:10)
    from huggingface_hub import PyTorchModelHubMixin
except Exception:  # pragma: no cover
    class PyTorchModelHubMixin:  # type: ignore
        pass

from . import scene as SC          # not "scene": the scene functions take an argument of that name
from . import torch_parts as TP
from .geometry import _is_int
from .params import AggregatorParams, CameraHeadParams, Component, DPTParams, init_parameters

_RESNET_MEAN = (0.485, 0.456, 0.406)   # reference models/aggregator.py:22-23
_RESNET_STD = (0.229, 0.224, 0.225)
_HEADS = ("camera_head", "depth_head", "point_head")
_DPT_HEADS = (("depth_head", 0), ("point_head", 1))          # name, head_act (exp / inverse-log)


def chunk_schedule(S: int, chunk: int, overlap: int) -> List[Tuple[int, int]]:
    """The view sets (start, end) of OmniVGGT.reconstruct over S views: one set when S <= chunk; else starts 0, step,
    2 step, ... (step = chunk - overlap) while start + chunk < S, then a last set at S - chunk.  Every set has chunk views
    and shares at least overlap views with the views before it."""
    if S <= chunk:
        return [(0, S)]
    out = [(a, a + chunk) for a in range(0, S - chunk, chunk - overlap)]
    return out + [(S - chunk, S)]


def chunk_index(idx: Optional[Sequence[int]], start: int, end: int) -> List[int]:
    """A view set's members of a list of global view indices, as indices into the set."""
    return [int(i) - start for i in (idx or []) if start <= int(i) < end]


class OmniVGGT(nn.Module, PyTorchModelHubMixin):
    def __init__(self, img_size: int = 518, patch_size: int = 14, embed_dim: int = 1024, *, depth: int = 24,
                 patch_embed: str = "dinov2_vitl14_reg", dino_depth: int = 24, dino_heads: int = 16,
                 num_register_tokens: int = 4, dpt_features: int = 256,
                 dpt_out_channels: Sequence[int] = (256, 512, 1024, 1024),
                 dpt_layers: Sequence[int] = (4, 11, 17, 23), camera_heads: int = 16, camera_trunk_depth: int = 4,
                 dino_backend: str = "ovg", dino_dtype: torch.dtype = torch.bfloat16, camera_backend: str = "ovg",
                 camera_dtype: torch.dtype = torch.bfloat16, dpt_dtype: str = "fp16",
                 use_cuda_graph: Optional[bool] = None, init_seed: Optional[int] = 0):
        super().__init__()
        self.img_size, self.patch_size, self.embed_dim = img_size, patch_size, embed_dim
        self.dpt_layers = tuple(dpt_layers)
        self.dino_backend = dino_backend   # "ovg": frozen patchifier on the libovg kernels; "torch": library kernels
        self.dino_dtype = dino_dtype
        self.camera_backend = camera_backend  # "ovg": camera head on the libovg runtime; "torch": library kernels
        self.camera_dtype = camera_dtype     # camera_backend="torch": precision of the weight matrices (fp32 selectable)
        # DPT heads: "fp16" (11-bit significand like the TF32 convolutions the reference's fp32 heads run with on a GPU; stores
        # saturate at +-65504) or "bf16" (8-bit significand, fp32 exponent range).  Same speed; see DESIGN.md section 2.
        assert dpt_dtype in ("fp16", "bf16")
        self.dpt_dtype = dpt_dtype
        # replay the ~1000 kernel launches of a forward from a CUDA graph once a shape has been seen twice
        self.use_cuda_graph = (os.environ.get("OVG_CUDA_GRAPH", "1") != "0") if use_cuda_graph is None else use_cuda_graph
        self._graphs = {}
        self.max_graphs = 8                 # captured input signatures kept (least recently used one is dropped)
        self.head_streams = os.environ.get("OVG_HEAD_STREAMS", "1") != "0"   # camera / depth / point heads on 3 streams
        self._streams = None
        pe = "conv" if "conv" in patch_embed else "dino"
        self.aggregator = AggregatorParams(img_size, patch_size, embed_dim, depth, 64, num_register_tokens, pe,
                                           dino_depth, dino_heads)
        self.camera_head = CameraHeadParams(2 * embed_dim, camera_trunk_depth, camera_heads)
        self.point_head = DPTParams(2 * embed_dim, 4, dpt_features, list(dpt_out_channels))   # inv_log / expp1
        self.depth_head = DPTParams(2 * embed_dim, 2, dpt_features, list(dpt_out_channels))   # exp / expp1
        self.register_buffer("_resnet_mean", torch.tensor(_RESNET_MEAN).view(1, 1, 3, 1, 1), persistent=False)
        self.register_buffer("_resnet_std", torch.tensor(_RESNET_STD).view(1, 1, 3, 1, 1), persistent=False)
        if init_seed is not None:
            init_parameters(self, init_seed, dezero=False)
        self._engine = None
        self._cp = None                     # ContextParallel state (enable_context_parallel)
        object.__setattr__(self, "_dino_lp", None)   # low-precision replica of the frozen patchifier (lazy, not in state_dict)

    # ---------------------------------------------------------------------------------------------- packing
    def randomize_(self, seed: int = 0, dezero: bool = True) -> "OmniVGGT":
        """Synthetic weights on the current device (benchmarks / smoke test; there is no checkpoint offline)."""
        init_parameters(self, seed, dezero)
        self._invalidate()
        return self

    def _invalidate(self):
        self._engine = None
        self._graphs = {}
        object.__setattr__(self, "_dino_lp", None)
        TP.clear_lp_cache(self)

    def _load_from_state_dict(self, *a, **k):  # invalidate packed weights on any (re)load
        self._invalidate()
        return super()._load_from_state_dict(*a, **k)

    def load_state_dict(self, *a, **k):
        self._invalidate()
        return super().load_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self._invalidate()
        return super()._apply(fn, *a, **k)

    def __setattr__(self, name, value):
        # the submodules are callable (params.Component): each holds a weak reference to the model that owns it, kept out of
        # parameters() / state_dict() / _modules.  A head set to None is skipped (omnivggt.py:46,:51,:58); the packed weights and
        # the captured graphs of the old set of heads go.
        if isinstance(value, Component):
            object.__setattr__(value, "_owner", weakref.ref(self))
        super().__setattr__(name, value)
        if name in _HEADS and "_engine" in self.__dict__:
            self._invalidate()

    def __setstate__(self, state):        # copy.deepcopy / pickle: the copies' components point at the copy
        super().__setstate__(state)
        for m in self.children():
            if isinstance(m, Component):
                object.__setattr__(m, "_owner", weakref.ref(self))

    def _dpt_heads(self):
        return [(name, act) for name, act in _DPT_HEADS if getattr(self, name) is not None]

    def _dino_module(self):
        """The frozen patchifier in ``dino_dtype``: a cached cast of the fp32 master weights (no per-call casts)."""
        pe = self.aggregator.patch_embed
        if self.dino_dtype == torch.float32:
            return pe
        if self._dino_lp is None:
            import copy
            lp = copy.deepcopy(pe).to(self.dino_dtype)
            object.__setattr__(self, "_dino_lp", lp)          # plain attribute: keep it out of parameters()/state_dict()
        return self._dino_lp

    def engine(self):
        """Repack weights into kernel layouts (bf16, K-major, folded LayerNorm affines) on first use."""
        if self._engine is None:
            from .engine import Engine          # imports the CUDA library; fails loudly if it is missing
            if next(self.parameters()).device.type != "cuda":
                raise RuntimeError("OmniVGGT (H100 engine) has no CPU path: move the module to a CUDA device")
            self._engine = Engine(self)
        return self._engine

    # ---------------------------------------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, images: torch.Tensor, extrinsics: torch.Tensor = None, intrinsics: torch.Tensor = None,
                depth: torch.Tensor = None, mask: torch.Tensor = None, depth_gt_index: list = None,
                camera_gt_index: list = None) -> Dict[str, object]:
        images, depth_idx, cam_idx = self._check_inputs(images, extrinsics, intrinsics, depth, mask, depth_gt_index,
                                                        camera_gt_index)
        eng = self.engine()
        args = (images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx)
        if self.use_cuda_graph and images.is_cuda and not torch.cuda.is_current_stream_capturing():
            return self._forward_graphed(eng, *args)
        return self._forward_impl(eng, *args)

    def _check_inputs(self, images, extrinsics, intrinsics, depth, mask, depth_gt_index, camera_gt_index):
        if images.dim() == 4:
            images = images.unsqueeze(0)
        B, S, Cin, H, W = images.shape
        if Cin != 3:
            raise ValueError(f"Expected 3 input channels, got {Cin}")                 # omnivggt_aggregator.py:139-140
        assert H % self.patch_size == 0, f"Input image height {H} is not a multiple of patch height {self.patch_size}"
        assert W % self.patch_size == 0, f"Input image width {W} is not a multiple of patch width: {self.patch_size}"
        # The fused RoPE epilogue holds 64 positions per axis (patch rows / columns + 1), so 63 patches = 882 px per side.
        # Refused here, before the DINOv2 patchifier or any other kernel runs, for every entry point that reaches the aggregator.
        limit = 63 * self.patch_size
        if max(H, W) > limit:
            raise ValueError(f"{H}x{W} input: at most {limit} px per side (the fused RoPE epilogue holds 64 positions per axis)")
        depth_idx = list(depth_gt_index) if depth_gt_index is not None else []
        cam_idx = list(camera_gt_index) if camera_gt_index is not None else []
        if len(depth_idx):
            assert depth is not None and mask is not None, "depth_gt_index given without depth / mask"
            assert tuple(depth.shape[:4]) == tuple(mask.shape), "mask and depth must have the same first four dimensions"
        if len(cam_idx):
            assert extrinsics is not None and intrinsics is not None, "camera_gt_index given without cameras"
        return images, depth_idx, cam_idx

    # ---------------------------------------------------------------------------------------------- context parallelism
    def enable_context_parallel(self, group=None) -> "OmniVGGT":
        """Shard the VIEWS of one scene over the ranks of a torch.distributed group on one node (SURVEY.md section 8f rank 2).
        Every rank then calls forward() with the SAME full inputs (B = 1, S divisible by the world size) and gets the dense
        predictions of ITS views (``view_range``) plus the pose encodings of all views.  See context_parallel.py."""
        from .context_parallel import ContextParallel
        self._cp = ContextParallel(next(self.parameters()).device, group)
        return self

    @staticmethod
    def _put_dpt(out, name, preds, conf, B, S, H, W):
        key = "depth" if name == "depth_head" else "world_points"
        out[key] = preds.view(B, S, H, W, preds.shape[-1])
        out[key + "_conf"] = conf.view(B, S, H, W)

    # ---------------------------------------------------------------------------------------------- components
    # model.aggregator(...), model.camera_head(...), model.depth_head(...) and model.point_head(...) take the reference's
    # arguments (params.Component) and land here.  They run eagerly (no CUDA graph) on one GPU.
    def _component_engine(self):
        if self._cp is not None:
            raise RuntimeError("the component calls (aggregator / camera_head / depth_head / point_head) run on one GPU; "
                               "under enable_context_parallel() call the model itself")
        return self.engine()

    @torch.no_grad()
    def _call_aggregator(self, images, extrinsics, intrinsics, depth, mask, depth_gt_index, camera_gt_index
                         ) -> Tuple[List[torch.Tensor], int]:
        """All ``depth`` layers in fp32 [B, S, T, 2C] (frame half | global half) and patch_start_idx = 1 + registers, as
        ZeroAggregator.forward returns them (omnivggt_aggregator.py:248-256).  Same patchifier, injection and kernels as
        forward(); the layers are written by the snapshot pass of the aggregator."""
        images, depth_idx, cam_idx = self._check_inputs(images, extrinsics, intrinsics, depth, mask, depth_gt_index,
                                                        camera_gt_index)
        eng = self._component_engine()
        B, S, _, H, W = images.shape
        T = (H // self.patch_size) * (W // self.patch_size) + eng.R + 1
        layers = [torch.empty(B, S, T, 2 * eng.C, device=eng.device, dtype=torch.float32) for _ in range(eng.depth)]
        self._aggregate(eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx, slots=False, layers=layers)
        return layers, 1 + eng.R

    @torch.no_grad()
    def _call_dpt(self, head, tokens, images, patch_start_idx, frames_chunk_size=8):
        """DPTHead.forward (dpt_head.py:128-183) on the layers ``dpt_layers`` of any fp32 token list [B, S, T, 2C] with
        T = patches + patch_start_idx; ``images`` gives H and W only.  The first LayerNorm reads the fp32 tokens and rounds them
        to bf16 as the aggregator's own snapshot does, so the output equals forward()'s bit for bit on this aggregator's tokens.
        Frames are chunked over B * S (the reference chunks each scene's S; every frame's result is chunk independent)."""
        eng = self._component_engine()
        name, act = next((n, a) for n, a in _DPT_HEADS if self._modules.get(n) is head)
        B, S, _, H, W = images.shape
        K = B * S
        T = (H // self.patch_size) * (W // self.patch_size) + patch_start_idx
        want = (B, S, T, 2 * eng.C)
        layers = {}
        for i in self.dpt_layers:
            t = tokens[i]
            if tuple(t.shape) != want:
                raise ValueError(f"{name}: layer {i} has shape {tuple(t.shape)}, expected {want} for {H}x{W} images")
            layers[i] = t.to(device=eng.device, dtype=torch.float32).contiguous().view(K, T, 2 * eng.C)
        chunk = K if frames_chunk_size is None else int(frames_chunk_size)
        if chunk <= 0:
            raise ValueError("frames_chunk_size must be positive")
        eng.warm_tables(H, W)
        preds, conf = eng.dpt(name, layers, self.dpt_layers, K, H, W, head_act=act, chunk=chunk, nspecial=patch_start_idx)
        return preds.view(B, S, H, W, preds.shape[-1]), conf.view(B, S, H, W)

    @torch.no_grad()
    def _call_camera(self, tokens, num_iterations=4) -> List[torch.Tensor]:
        """CameraHead.forward (camera_head.py:83-103): the camera tokens tokens[-1][:, :, 0]."""
        eng = self._component_engine()
        last = tokens[-1]
        B, S = last.shape[:2]
        cam = last[:, :, 0].to(device=eng.device, dtype=torch.float32).contiguous()
        if eng.h_cam is not None:
            return eng.camera_head(cam.view(B * S, -1), B, S, iters=num_iterations)
        return TP.camera_head(self.camera_head, cam, iters=num_iterations, dtype=self.camera_dtype)

    # ---------------------------------------------------------------------------------------------- post-processing (scene.py)
    postprocess = staticmethod(SC.postprocess)
    sky_mask = staticmethod(SC.sky_mask)
    point_cloud = staticmethod(SC.point_cloud)
    mesh = staticmethod(SC.mesh)
    matches = staticmethod(SC.matches)
    tracks = staticmethod(SC.tracks)
    bundle_adjust = staticmethod(SC.bundle_adjust)
    fused_mesh = staticmethod(SC.fused_mesh)
    _kept_views = staticmethod(SC._kept_views)          # their shared helpers, reached from the class as before
    _align = staticmethod(SC._align)

    # ---------------------------------------------------------------------------------------------- long captures
    @torch.no_grad()
    def reconstruct(self, images: torch.Tensor, extrinsics: torch.Tensor = None, intrinsics: torch.Tensor = None,
                    depth: torch.Tensor = None, mask: torch.Tensor = None, depth_gt_index: list = None,
                    camera_gt_index: list = None, *, chunk: int = 24, overlap: int = 8, source: str = "depth",
                    conf_percent: float = 50.0) -> Dict[str, object]:
        """One scene longer than one forward, as overlapping view sets merged into the frame and scale of the first.

        Views are taken in the given order (permute them first for an unordered collection, e.g. by
        ``geometry.compute_ranking``).  The view sets are ``chunk_schedule(S, chunk, overlap)``: each has ``chunk`` views (so
        every forward replays one CUDA graph) and shares at least ``overlap`` views with the views before it.
        ``depth_gt_index`` / ``camera_gt_index`` hold global view indices; each view set gets its members, re-indexed.

        Per view set: the forward on its views, then the cameras decoded and the depth unprojected as ``postprocess`` does.
        The first set is kept as it is.  Each later set is aligned by the similarity (libovg ovg_sim3_estimate) that maps its
        points of the views it shares with the merge onto the merged points of those views, over the pixels kept on both
        sides by point_cloud's rule (conf >= percentile(conf over those views, conf_percent) and conf > 1e-5), with
        ``source`` selecting the points as in ``point_cloud``.  Its new views are then mapped into the merge (libovg
        ovg_sim3_apply: points, depth and extrinsics in fp64, rounded once; intrinsics and confidences copied).  A view kept
        by several sets keeps the outputs of the first.  Only one set's raw outputs are held at a time.

        Returns a dict with B = 1 that ``point_cloud``, ``mesh``, ``matches`` and ``sky_mask`` take as it is: ``images``,
        ``extrinsic``, ``intrinsic``, ``depth``, ``depth_conf``, ``world_points_from_depth`` and, with the point head,
        ``world_points`` / ``world_points_conf``; ``chunks`` [(start, end)]; ``sim3`` fp64 [n_chunks, 4, 4] mapping each set
        into the first set's frame; ``align_pairs`` and ``align_rmse`` fp64 [n_chunks] (0 for the first set).  ``pose_enc``
        is not returned: it is normalised per view set.  The alignment statistics are read once per set boundary, and a
        degenerate overlap raises ValueError naming the set and its views.  Errors accumulate along the chain of sets (no
        loop closure)."""
        if self._cp is not None:
            raise RuntimeError("reconstruct runs its view sets on one GPU; under enable_context_parallel() call the model itself")
        if images.dim() == 4:
            images = images.unsqueeze(0)
        if images.dim() != 5 or images.shape[0] != 1:
            raise ValueError(f"reconstruct takes one scene (B = 1), got images of shape {tuple(images.shape)}")
        for name, v in (("chunk", chunk), ("overlap", overlap)):
            if not _is_int(v):
                raise ValueError(f"{name} must be an integer, got {v!r}")
        if chunk < 2:
            raise ValueError(f"chunk must be >= 2, got {chunk}")
        if not 1 <= overlap < chunk:
            raise ValueError(f"overlap must be in [1, chunk - 1 = {chunk - 1}], got {overlap}")
        if source not in ("depth", "pointmap"):
            raise ValueError(f"source must be 'depth' or 'pointmap', got {source!r}")
        if source == "pointmap" and self.point_head is None:
            raise ValueError("source='pointmap' needs the point head (it is set to None)")
        if self.camera_head is None or self.depth_head is None:
            raise ValueError("reconstruct needs the camera head and the depth head")
        if not 0.0 <= conf_percent <= 100.0:
            raise ValueError("conf_percent must be in [0, 100]")
        S, H, W = images.shape[1], images.shape[-2], images.shape[-1]
        for name, idx in (("depth_gt_index", depth_gt_index), ("camera_gt_index", camera_gt_index)):
            if any(not 0 <= int(i) < S for i in (idx or [])):
                raise IndexError(f"{name} {list(idx)} out of range for {S} views")
        chunks = chunk_schedule(S, chunk, overlap)
        merged: Dict[str, torch.Tensor] = {}
        sims, stats_all = [], []
        for k, (a, b) in enumerate(chunks):
            di, ci = chunk_index(depth_gt_index, a, b), chunk_index(camera_gt_index, a, b)
            part = (lambda t: None if t is None else t[:, a:b])
            raw = self(images[:, a:b], part(extrinsics), part(intrinsics), part(depth), part(mask), depth_gt_index=di,
                       camera_gt_index=ci)
            n = b - a
            ext, intr, world = SC.decode_cameras(raw["pose_enc"][0], raw["depth"][0], H, W)
            r = {"extrinsic": ext, "intrinsic": intr, "depth": raw["depth"][0], "depth_conf": raw["depth_conf"][0],
                 "world_points_from_depth": world}
            if "world_points" in raw:
                r["world_points"], r["world_points_conf"] = raw["world_points"][0], raw["world_points_conf"][0]
            del raw
            if k == 0:
                dev = ext.device
                merged = {key: torch.empty((1, S) + tuple(v.shape[1:]), device=dev, dtype=torch.float32) for key, v in r.items()}
                for key, v in r.items():
                    merged[key][0, :n].copy_(v)
                sims.append(torch.eye(4, device=dev, dtype=torch.float64))
                stats_all.append(torch.zeros(4, device=dev, dtype=torch.float64))
                continue
            sim3, stats = self._merge_view_set(merged, r, k, a, chunks[k - 1][1], b, source, conf_percent)
            sims.append(sim3)
            stats_all.append(stats)
        stats = torch.stack(stats_all)
        merged.update(images=images, chunks=chunks, sim3=torch.stack(sims), align_pairs=stats[:, 0].clone(),
                      align_rmse=stats[:, 2].clone())
        return merged

    @staticmethod
    def _merge_view_set(merged: Dict[str, torch.Tensor], r: Dict[str, torch.Tensor], k: int, a: int, n0: int, b: int,
                        source: str, conf_percent: float):
        """Aligns view set k (views a..b-1, outputs r in its own frame) on its views a..n0-1 that are merged already and
        writes its views n0..b-1 into the merged tensors.  Returns (sim3, stats) on the device; the status is read here."""
        from . import geometry, ops
        pkey, ckey = ("world_points_from_depth", "depth_conf") if source == "depth" else ("world_points", "world_points_conf")
        m_src, _, _ = ops.conf_percentile_mask(r[ckey][:n0 - a].contiguous(), conf_percent, 1e-5)
        m_dst, _, _ = ops.conf_percentile_mask(merged[ckey][0, a:n0].contiguous(), conf_percent, 1e-5)
        sim3, stats = ops.sim3_estimate(r[pkey][:n0 - a].reshape(-1, 3), merged[pkey][0, a:n0].reshape(-1, 3),
                                        (m_src & m_dst).view(-1))
        status = int(ops.host_read(stats)[1])
        if status:
            raise ValueError(f"view set {k} (views {a}..{b - 1}) cannot be aligned on its shared views {a}..{n0 - 1}: "
                             f"{geometry.SIM3_STATUS[status]}")
        new = slice(n0 - a, b - a)
        H, W = r["depth"].shape[1:3]
        ops.sim3_apply(sim3, b - n0, H * W,
                       points=[(r[key][new], merged[key][0, n0:b]) for key in ("world_points_from_depth", "world_points")
                               if key in r],
                       depth=(r["depth"][new], merged["depth"][0, n0:b]),
                       ext=(r["extrinsic"][new], merged["extrinsic"][0, n0:b]))
        for key in ("intrinsic", "depth_conf", "world_points_conf"):
            if key in r:
                merged[key][0, n0:b].copy_(r[key][new])
        return sim3, stats

    # ---------------------------------------------------------------------------------------------- CUDA graph replay
    def _forward_graphed(self, eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx):
        """Same computation, launched from a captured CUDA graph (a forward is >1000 kernel launches; issuing them from
        Python costs about as much host time as the GPU needs to run them).  A graph is captured the third time a
        (shape, index-list) signature is seen; inputs are copied into static buffers, outputs are cloned."""
        need_c, need_d = len(cam_idx) > 0, len(depth_idx) > 0
        def sig(t):
            return None if t is None else (tuple(t.shape), t.dtype)
        heads = tuple(getattr(self, n) is not None for n in _HEADS)
        key = (self._cp is not None, sig(images), tuple(depth_idx), tuple(cam_idx), sig(extrinsics) if need_c else None,
               sig(intrinsics) if need_c else None, sig(depth) if need_d else None, sig(mask) if need_d else None, heads)
        ent = self._graphs.pop(key, None)
        if ent is None:
            ent = {"calls": 0, "graph": None}
            while len(self._graphs) >= self.max_graphs:     # LRU: a graph owns static inputs + a private output pool
                self._graphs.pop(next(iter(self._graphs)))
        self._graphs[key] = ent                             # most recently used last
        ent["calls"] += 1
        if ent["graph"] is None and (ent["calls"] < 3 or ent.get("failed")):
            return self._forward_impl(eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx)
        dyn = [images, extrinsics if need_c else None, intrinsics if need_c else None, depth if need_d else None,
               mask if need_d else None]
        if ent["graph"] is None or ent["ws_version"] != eng.ws.version:
            try:
                static = [None if t is None else t.detach().clone() for t in dyn]
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):      # allocator warm-up on a side stream, as the capture API requires
                    self._forward_impl(eng, *static, depth_idx, cam_idx)
                torch.cuda.current_stream().wait_stream(s)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    out = self._forward_impl(eng, *static, depth_idx, cam_idx)
                ent.update(graph=g, static=static, out=out, ws_version=eng.ws.version)
            except torch.cuda.OutOfMemoryError as ex:
                # the only failure that is a property of the call, not a bug: the private pool of one more graph does not fit.
                # Everything else (a capture-illegal operation, a kernel error) propagates.
                ent["failed"] = True
                ent["graph"] = None
                warnings.warn(f"OmniVGGT: no memory for another CUDA graph ({ex}); this signature keeps eager launches")
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                return self._forward_impl(eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx)
        for st, t in zip(ent["static"], dyn):
            if st is not None:
                st.copy_(t)
        ent["graph"].replay()
        out = ent["out"]
        res = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in out.items() if k not in ("images", "pose_enc_list")}
        if "pose_enc_list" in out:
            res["pose_enc_list"] = [t.clone() for t in out["pose_enc_list"]]
            res["pose_enc"] = res["pose_enc_list"][-1]
        res["images"] = images if "view_range" not in out else images[:, out["view_range"][0]:out["view_range"][1]]
        return res

    def _camera(self, eng, cam_tokens, B, S):
        if eng.h_cam is not None:
            return eng.camera_head(cam_tokens, B, S)
        return TP.camera_head(self.camera_head, cam_tokens.view(B, S, -1), dtype=self.camera_dtype)

    def _aggregate(self, eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx, slots=True, layers=None, sl=None):
        """Patchifier, camera / depth injection and the aggregator on the views ``sl`` of each scene (default: all of them;
        this rank's under context parallelism): (bf16 slots of the kept layers, fp32 camera tokens [B*S, 2C] of ALL S views).
        Under context parallelism the camera tokens are the ones every rank gathered (cp.cam_all)."""
        B, S, Cin, H, W = images.shape
        ag = self.aggregator
        cp = self._cp
        sl = slice(0, S) if sl is None else sl
        n = sl.stop - sl.start
        K = B * n

        # ---- frozen patchifier (PyTorch): normalise, DINOv2 / conv patch embed       (omnivggt_aggregator.py:143-150)
        if eng.dino is not None:
            P = (H // self.patch_size) * (W // self.patch_size)
            pos = TP.dino_pos_embed(ag.patch_embed, P, H, W, self.patch_size).float()
            patch = eng.dino_patchify(images[:, sl].float().view(K, Cin, H, W), pos, _RESNET_MEAN, _RESNET_STD)
        elif cp is not None:
            raise RuntimeError("context parallelism runs the DINOv2 patchifier on the libovg runtime (dino_backend='ovg')")
        else:
            img = ((images.float() - self._resnet_mean) / self._resnet_std).view(K, Cin, H, W)
            if hasattr(ag.patch_embed, "blocks"):
                patch = TP.dino_patchify(self._dino_module(), img, self.patch_size, self.dino_dtype)
            else:
                pe = ag.patch_embed.proj
                patch = torch.nn.functional.conv2d(img, pe.weight, pe.bias, stride=self.patch_size).flatten(2).transpose(1, 2)
            patch = patch.float().contiguous()

        # ---- aux cameras -> pose encoding -> 25 injection vectors (tiny fp32 host math)  (:158-182,:273-287)
        # The pose normalisation is global over the selected views of a scene (omnivggt_aggregator.py:85-105), and the inputs
        # are a few hundred bytes per view, so the vectors are computed for all S views and the views of ``sl`` kept.
        pose = None
        rows = None
        if len(cam_idx):
            ci = eng.cached(("cam_idx", tuple(cam_idx)), lambda: torch.tensor(cam_idx))
            rows = eng.cached(("cam_rows", B, S, tuple(cam_idx)),
                              lambda: (torch.arange(B)[:, None] * S + torch.tensor(cam_idx)[None]).reshape(-1))
            pose = TP.aux_pose_encoding(extrinsics.index_select(1, ci), intrinsics.index_select(1, ci), H, W)
        inj = TP.injection_vectors(eng.inj_pack, pose, cam_idx, B, S, rows)
        inj = inj.view(-1, B, S, inj.shape[-1])[:, :, sl].reshape(-1, K, inj.shape[-1])      # a view when sl is every view

        # ---- hot path: aggregator on libovg.  Under context parallelism depth / mask are the full tensors and depth_idx holds
        # scene indices: the masked-mean normalisation of the depth modality is over all selected views of the scene.
        keep = set(self.dpt_layers)
        slots, cam_out = eng.aggregate(patch, inj, depth, mask, depth_idx, B, n, H, W, keep, cp=cp, views_total=S, slots=slots,
                                       layers=layers)
        return slots, (cp.cam_all if cp is not None else cam_out)

    def _forward_impl(self, eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx):
        B, S, Cin, H, W = images.shape
        sl = slice(0, S)
        if self._cp is not None:
            if B != 1:
                raise ValueError("context parallelism shards the views of ONE scene (B = 1); use scene-level data parallelism for "
                                 "batches")
            v0, n = self._cp.local_views(S)
            sl = slice(v0, v0 + n)
        n = sl.stop - sl.start                    # views of each scene with dense outputs
        K = B * n
        heads = self._dpt_heads()                 # the heads set to None are skipped, as the reference does (omnivggt.py:46-62)
        cam_on = self.camera_head is not None
        slots, cam_tokens = self._aggregate(eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx, slots=bool(heads),
                                            sl=sl)

        # ---- heads.  The camera head and the two DPT heads only read the aggregator outputs: they run on three streams
        # (forked / joined with events, also inside a captured CUDA graph) so that their many small kernels -- 19^2 / 37^2
        # feature maps, M = 8 GEMVs -- share the 132 SMs instead of running one after the other.
        predictions: Dict[str, object] = {}
        eng.warm_tables(H, W)
        outs = {name: eng.dpt_alloc(name, K, H, W) for name, _ in heads}
        pose_list = None

        def dpt(name, act):
            eng.dpt(name, slots, self.dpt_layers, K, H, W, head_act=act, out=outs[name])

        main = torch.cuda.current_stream() if images.is_cuda else None
        if main is not None and self._cp is None and self.head_streams and cam_on + len(heads) > 1:
            if self._streams is None:
                self._streams = (torch.cuda.Stream(), torch.cuda.Stream())
            side = list(self._streams)
            fork = torch.cuda.Event()
            fork.record(main)
            work = ([("camera", None)] if cam_on else []) + heads[::-1]
            for name, act in work[:-1]:                  # the camera head and the point head on side streams
                s = side.pop(0)
                s.wait_event(fork)
                with torch.cuda.stream(s):
                    if name == "camera":
                        pose_list = self._camera(eng, cam_tokens, B, S)
                    else:
                        dpt(name, act)
            name, act = work[-1]                         # the depth head (or the last head present) on the main stream
            if name == "camera":
                pose_list = self._camera(eng, cam_tokens, B, S)
            else:
                dpt(name, act)
            for s in self._streams[:len(work) - 1]:
                main.wait_stream(s)
        else:
            if cam_on:
                pose_list = self._camera(eng, cam_tokens, B, S)
            for name, act in heads:
                dpt(name, act)
        if cam_on:
            predictions["pose_enc"] = pose_list[-1]
            predictions["pose_enc_list"] = pose_list
        for name, _ in heads:
            self._put_dpt(predictions, name, *outs[name], B, n, H, W)
        predictions["images"] = images
        if self._cp is not None:
            predictions["images"], predictions["view_range"] = images[:, sl], (sl.start, sl.stop)
        return predictions
