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
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

try:  # keep from_pretrained / save_pretrained like the reference (omnivggt.py:3,:10)
    from huggingface_hub import PyTorchModelHubMixin
except Exception:  # pragma: no cover
    class PyTorchModelHubMixin:  # type: ignore
        pass

from . import torch_parts as TP
from .params import AggregatorParams, CameraHeadParams, DPTParams, init_parameters

_RESNET_MEAN = (0.485, 0.456, 0.406)   # reference models/aggregator.py:22-23
_RESNET_STD = (0.229, 0.224, 0.225)


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
        if images.dim() == 4:
            images = images.unsqueeze(0)
        B, S, Cin, H, W = images.shape
        if Cin != 3:
            raise ValueError(f"Expected 3 input channels, got {Cin}")                 # omnivggt_aggregator.py:139-140
        assert H % self.patch_size == 0, f"Input image height {H} is not a multiple of patch height {self.patch_size}"
        assert W % self.patch_size == 0, f"Input image width {W} is not a multiple of patch width: {self.patch_size}"
        depth_idx = list(depth_gt_index) if depth_gt_index is not None else []
        cam_idx = list(camera_gt_index) if camera_gt_index is not None else []
        if len(depth_idx):
            assert depth is not None and mask is not None, "depth_gt_index given without depth / mask"
            assert tuple(depth.shape[:4]) == tuple(mask.shape), "mask and depth must have the same first four dimensions"
        if len(cam_idx):
            assert extrinsics is not None and intrinsics is not None, "camera_gt_index given without cameras"
        eng = self.engine()
        args = (images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx)
        impl = self._forward_cp if self._cp is not None else self._forward_impl
        if self.use_cuda_graph and images.is_cuda and not torch.cuda.is_current_stream_capturing():
            return self._forward_graphed(eng, impl, *args)
        return impl(eng, *args)

    # ---------------------------------------------------------------------------------------------- context parallelism
    def enable_context_parallel(self, group=None) -> "OmniVGGT":
        """Shard the VIEWS of one scene over the ranks of a torch.distributed group on one node (SURVEY.md section 8f rank 2).
        Every rank then calls forward() with the SAME full inputs (B = 1, S divisible by the world size) and gets the dense
        predictions of ITS views (``view_range``) plus the pose encodings of all views.  See context_parallel.py."""
        from .context_parallel import ContextParallel
        self._cp = ContextParallel(next(self.parameters()).device, group)
        return self

    def _forward_cp(self, eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx):
        cp = self._cp
        B, S, Cin, H, W = images.shape
        if B != 1:
            raise ValueError("context parallelism shards the views of ONE scene (B = 1); use scene-level data parallelism for batches")
        v0, n = cp.local_views(S)
        sl = slice(v0, v0 + n)
        ag = self.aggregator
        if eng.dino is None:
            raise RuntimeError("context parallelism runs the DINOv2 patchifier on the libovg runtime (dino_backend='ovg')")
        P = (H // self.patch_size) * (W // self.patch_size)
        pos = TP.dino_pos_embed(ag.patch_embed, P, H, W, self.patch_size).float()
        patch = eng.dino_patchify(images[0, sl].float().contiguous(), pos, _RESNET_MEAN, _RESNET_STD)
        # camera aux: pose normalisation is global over the selected views (omnivggt_aggregator.py:85-105), the inputs are a
        # few hundred bytes per view and replicated, so every rank computes all injection vectors and keeps its columns
        pose = rows = None
        if len(cam_idx):
            ci = eng.cached(("cam_idx", tuple(cam_idx)), lambda: torch.tensor(cam_idx))
            rows = eng.cached(("cam_rows", 1, S, tuple(cam_idx)), lambda: torch.tensor(cam_idx))
            pose = TP.aux_pose_encoding(extrinsics.index_select(1, ci), intrinsics.index_select(1, ci), H, W)
        inj = TP.injection_vectors(eng.inj_pack, pose, cam_idx, 1, S, rows)[:, sl].contiguous()
        # depth aux: full tensors + scene indices (the masked-mean normalisation is over all selected views of the scene)
        slots, cam_loc = eng.aggregate(patch, inj, depth, mask, depth_idx, 1, n, H, W, set(self.dpt_layers), cp=cp, views_total=S)
        pose_list = self._camera(eng, cp.cam_all, 1, S)            # [S, 2C] gathered by peer stores: the camera head attends across all views
        eng.warm_tables(H, W)
        d_out = eng.dpt("depth_head", slots, self.dpt_layers, n, H, W, head_act=0)
        p_out = eng.dpt("point_head", slots, self.dpt_layers, n, H, W, head_act=1)
        return {"pose_enc": pose_list[-1], "pose_enc_list": pose_list, "depth": d_out[0].view(1, n, H, W, 1),
                "depth_conf": d_out[1].view(1, n, H, W), "world_points": p_out[0].view(1, n, H, W, 3),
                "world_points_conf": p_out[1].view(1, n, H, W), "images": images[:, sl], "view_range": (v0, v0 + n)}

    # ---------------------------------------------------------------------------------------------- post-processing
    @torch.no_grad()
    def postprocess(self, predictions: Dict[str, object], conf_percent: float = 50.0, use_point_map: bool = False
                    ) -> Dict[str, object]:
        """What reference inference.py does on the host right after the forward, on the device (libovg kernels):
        ``extrinsic`` / ``intrinsic`` from ``pose_enc`` (inference.py:360-365 -> utils/pose_enc.py:65-130),
        ``world_points_from_depth`` by unprojecting the predicted depth with the predicted cameras (visual_util.py:42-73 ->
        utils/geometry.py:151-264), and the confidence filter of the viewer (inference.py:132-133): ``conf_mask`` =
        conf >= percentile(conf, conf_percent) & conf > 0.1 with ``conf_threshold`` / ``conf_kept``, over
        ``world_points_conf`` if ``use_point_map`` else ``depth_conf`` (inference.py:95-100).  Adds the keys in place."""
        from . import ops
        pose = predictions["pose_enc"]
        H, W = predictions["images"].shape[-2:]
        B, S = pose.shape[:2]
        ext, intr, c2w = ops.pose_decode(pose.float(), H, W)
        predictions["extrinsic"], predictions["intrinsic"] = ext, intr
        depth = predictions["depth"].float().reshape(B * S, H, W)
        world = ops.unproject_depth(depth, intr.view(B * S, 3, 3), c2w.view(B * S, 3, 4), H, W)
        predictions["world_points_from_depth"] = world.view(B, S, H, W, 3)
        conf = predictions["world_points_conf" if use_point_map else "depth_conf"].float()
        mask, thr, cnt = ops.conf_percentile_mask(conf, conf_percent, 0.1)
        predictions["conf_mask"], predictions["conf_threshold"], predictions["conf_kept"] = mask.bool(), thr, cnt
        return predictions

    @staticmethod
    @torch.no_grad()
    def point_cloud(predictions: Dict[str, object], *, source: str = "depth", conf_percent: float = 50.0,
                    conf_floor: float = 1e-5, frame: Optional[int] = None, mask_black_bg: bool = False,
                    mask_white_bg: bool = False, scene: int = 0) -> Dict[str, torch.Tensor]:
        """The filtered, coloured point cloud of one scene, built on the device (libovg kernels).

        Replaces the host numpy of the reference's GLB export (visual_util.py:190-236,:320-358 predictions_to_glb) and
        viewer (inference.py:96-151).  ``source="depth"``: ``world_points_from_depth`` (computed here when ``postprocess``
        has not run) with ``depth_conf``, as ``--save_glb`` uses it; ``"pointmap"``: ``world_points`` with
        ``world_points_conf``.  ``frame``: keep only that view, selected before the percentile (visual_util.py:190-194).
        Kept: conf >= percentile(conf, conf_percent) (0 for conf_percent == 0, visual_util.py:206-207) and conf > conf_floor,
        minus black / white background pixels when asked.  ``conf_floor=0.1`` reproduces the viewer's initial mask
        (inference.py:132-133); its frame dropdown is ``cloud["frame"] == i`` on the ``frame=None`` cloud.

        Returns ``points`` fp32 [n,3], ``colors`` uint8 [n,3], ``frame`` int32 [n] (numpy boolean-indexing order),
        ``conf_threshold`` (0-d), ``center`` fp32 [3] (mean of all points of the selected views, inference.py:111),
        ``scale`` (0-d, ||p95 - p5||, 1.0 when nothing is kept) and ``align`` fp64 [4,4] = inv(E0) diag(1,-1,-1,1) R_y(180)
        with E0 the first selected camera (visual_util.py:320-341).  The kept count and E0 are the only device-to-host reads."""
        from . import ops
        if source not in ("depth", "pointmap"):
            raise ValueError(f"source must be 'depth' or 'pointmap', got {source!r}")
        if not 0.0 <= conf_percent <= 100.0:
            raise ValueError("conf_percent must be in [0, 100]")
        if conf_floor < 0.0:
            raise ValueError("conf_floor must be >= 0")        # the reference's floors are 1e-5 and 0.1

        def scene_of(t, trailing):                             # [B, S, ...] or [S, ...] -> [S, ...] of the scene
            return t[scene] if t.dim() == trailing + 2 else t

        images = scene_of(predictions["images"], 3).float()
        S, _, H, W = images.shape
        if "extrinsic" in predictions:
            ext = scene_of(predictions["extrinsic"], 2).float()
            c2w = None
        else:
            ext, intr, c2w = ops.pose_decode(scene_of(predictions["pose_enc"], 1).float().contiguous(), H, W)
        if source == "pointmap":
            points = scene_of(predictions["world_points"], 3)
            conf = scene_of(predictions["world_points_conf"], 2)
        else:
            if "world_points_from_depth" in predictions:
                points = scene_of(predictions["world_points_from_depth"], 3)
            else:
                if c2w is None:
                    ext, intr, c2w = ops.pose_decode(scene_of(predictions["pose_enc"], 1).float().contiguous(), H, W)
                depth = scene_of(predictions["depth"], 3).float().reshape(S, H, W)
                points = ops.unproject_depth(depth, intr, c2w, H, W)
            conf = scene_of(predictions["depth_conf"], 2)
        f0 = 0
        if frame is not None:
            if not 0 <= frame < S:
                raise IndexError(f"frame {frame} out of range for {S} views")
            f0 = frame
            images, points, conf = images[frame:frame + 1], points[frame:frame + 1], conf[frame:frame + 1]
        images = images.contiguous()
        points = points.float().contiguous()
        conf = conf.float().contiguous()
        F = images.shape[0]
        dev = images.device

        mask, thr, _ = ops.conf_percentile_mask(conf, conf_percent, conf_floor)
        if conf_percent == 0.0:
            thr = torch.zeros((), device=dev, dtype=torch.float32)   # same mask: conf > conf_floor >= 0 implies conf >= 0
        ws = ops.point_cloud_workspace(F * H * W, dev)
        cnt = ops.point_cloud_count(mask, images, ws, mask_black_bg, mask_white_bg)
        center = ops.point_cloud_center(points, ws)
        n = int(cnt.item())
        e0 = torch.eye(4, dtype=torch.float64)
        e0[:3, :4] = ext[f0].double().cpu()
        gl = torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0], dtype=torch.float64))
        rot_y = torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0], dtype=torch.float64))
        align = (torch.linalg.inv(e0) @ gl @ rot_y).to(dev)
        if n == 0:
            return {"points": torch.empty(0, 3, device=dev), "colors": torch.empty(0, 3, device=dev, dtype=torch.uint8),
                    "frame": torch.empty(0, device=dev, dtype=torch.int32), "conf_threshold": thr, "center": center,
                    "scale": torch.ones((), device=dev), "align": align}
        pts, cols, fr, xyz = ops.point_cloud_gather(points, mask, images, ws, n, mask_black_bg, mask_white_bg, f0)
        scale = ops.point_cloud_scale(xyz, n, ws)
        return {"points": pts, "colors": cols, "frame": fr, "conf_threshold": thr, "center": center, "scale": scale,
                "align": align}

    # ---------------------------------------------------------------------------------------------- CUDA graph replay
    def _forward_graphed(self, eng, impl, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx):
        """Same computation, launched from a captured CUDA graph (a forward is >1000 kernel launches; issuing them from
        Python costs about as much host time as the GPU needs to run them).  A graph is captured the third time a
        (shape, index-list) signature is seen; inputs are copied into static buffers, outputs are cloned."""
        need_c, need_d = len(cam_idx) > 0, len(depth_idx) > 0
        def sig(t):
            return None if t is None else (tuple(t.shape), t.dtype)
        key = (impl.__name__, sig(images), tuple(depth_idx), tuple(cam_idx), sig(extrinsics) if need_c else None,
               sig(intrinsics) if need_c else None, sig(depth) if need_d else None, sig(mask) if need_d else None)
        ent = self._graphs.pop(key, None)
        if ent is None:
            ent = {"calls": 0, "graph": None}
            while len(self._graphs) >= self.max_graphs:     # LRU: a graph owns static inputs + a private output pool
                self._graphs.pop(next(iter(self._graphs)))
        self._graphs[key] = ent                             # most recently used last
        ent["calls"] += 1
        if ent["graph"] is None and (ent["calls"] < 3 or ent.get("failed")):
            return impl(eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx)
        dyn = [images, extrinsics if need_c else None, intrinsics if need_c else None, depth if need_d else None,
               mask if need_d else None]
        if ent["graph"] is None or ent["ws_version"] != eng.ws.version:
            try:
                static = [None if t is None else t.detach().clone() for t in dyn]
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):      # allocator warm-up on a side stream, as the capture API requires
                    impl(eng, *static, depth_idx, cam_idx)
                torch.cuda.current_stream().wait_stream(s)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    out = impl(eng, *static, depth_idx, cam_idx)
                ent.update(graph=g, static=static, out=out, ws_version=eng.ws.version)
            except torch.cuda.OutOfMemoryError as ex:
                # the only failure that is a property of the call, not a bug: the private pool of one more graph does not fit.
                # Everything else (a capture-illegal operation, a kernel error) propagates.
                ent["failed"] = True
                ent["graph"] = None
                warnings.warn(f"OmniVGGT: no memory for another CUDA graph ({ex}); this signature keeps eager launches")
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                return impl(eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx)
        for st, t in zip(ent["static"], dyn):
            if st is not None:
                st.copy_(t)
        ent["graph"].replay()
        out = ent["out"]
        res = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in out.items() if k not in ("images", "pose_enc_list")}
        res["pose_enc_list"] = [t.clone() for t in out["pose_enc_list"]]
        res["pose_enc"] = res["pose_enc_list"][-1]
        res["images"] = images if "view_range" not in out else images[:, out["view_range"][0]:out["view_range"][1]]
        return res

    def _camera(self, eng, cam_tokens, B, S):
        if eng.h_cam is not None:
            return eng.camera_head(cam_tokens, B, S)
        return TP.camera_head(self.camera_head, cam_tokens.view(B, S, -1), dtype=self.camera_dtype)

    def _forward_impl(self, eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx):
        B, S, Cin, H, W = images.shape
        ag = self.aggregator
        K = B * S

        # ---- frozen patchifier (PyTorch): normalise, DINOv2 / conv patch embed       (omnivggt_aggregator.py:143-150)
        if eng.dino is not None:
            P = (H // self.patch_size) * (W // self.patch_size)
            pos = TP.dino_pos_embed(ag.patch_embed, P, H, W, self.patch_size).float()
            patch = eng.dino_patchify(images.float().view(K, Cin, H, W), pos, _RESNET_MEAN, _RESNET_STD)
        else:
            img = ((images.float() - self._resnet_mean) / self._resnet_std).view(K, Cin, H, W)
            if hasattr(ag.patch_embed, "blocks"):
                patch = TP.dino_patchify(self._dino_module(), img, self.patch_size, self.dino_dtype)
            else:
                pe = ag.patch_embed.proj
                patch = torch.nn.functional.conv2d(img, pe.weight, pe.bias, stride=self.patch_size).flatten(2).transpose(1, 2)
            patch = patch.float().contiguous()

        # ---- aux cameras -> pose encoding -> 25 injection vectors (tiny fp32 host math)  (:158-182,:273-287)
        pose = None
        rows = None
        if len(cam_idx):
            ci = eng.cached(("cam_idx", tuple(cam_idx)), lambda: torch.tensor(cam_idx))
            rows = eng.cached(("cam_rows", B, S, tuple(cam_idx)),
                              lambda: (torch.arange(B)[:, None] * S + torch.tensor(cam_idx)[None]).reshape(-1))
            pose = TP.aux_pose_encoding(extrinsics.index_select(1, ci), intrinsics.index_select(1, ci), H, W)
        inj = TP.injection_vectors(eng.inj_pack, pose, cam_idx, B, S, rows)

        # ---- hot path: aggregator on libovg
        keep = set(self.dpt_layers)
        slots, cam_tokens = eng.aggregate(patch, inj, depth, mask, depth_idx, B, S, H, W, keep)

        # ---- heads.  The camera head and the two DPT heads only read the aggregator outputs: they run on three streams
        # (forked / joined with events, also inside a captured CUDA graph) so that their many small kernels -- 19^2 / 37^2
        # feature maps, M = 8 GEMVs -- share the 132 SMs instead of running one after the other.
        predictions: Dict[str, object] = {}
        eng.warm_tables(H, W)
        d_out = eng.dpt_alloc("depth_head", K, H, W)
        p_out = eng.dpt_alloc("point_head", K, H, W)
        main = torch.cuda.current_stream() if images.is_cuda else None
        if main is not None and self.head_streams:
            if self._streams is None:
                self._streams = (torch.cuda.Stream(), torch.cuda.Stream())
            s_cam, s_pt = self._streams
            fork = torch.cuda.Event()
            fork.record(main)
            s_cam.wait_event(fork)
            s_pt.wait_event(fork)
            with torch.cuda.stream(s_cam):
                pose_list = self._camera(eng, cam_tokens, B, S)
            with torch.cuda.stream(s_pt):
                eng.dpt("point_head", slots, self.dpt_layers, K, H, W, head_act=1, out=p_out)
            eng.dpt("depth_head", slots, self.dpt_layers, K, H, W, head_act=0, out=d_out)
            main.wait_stream(s_cam)
            main.wait_stream(s_pt)
        else:
            pose_list = self._camera(eng, cam_tokens, B, S)
            eng.dpt("depth_head", slots, self.dpt_layers, K, H, W, head_act=0, out=d_out)
            eng.dpt("point_head", slots, self.dpt_layers, K, H, W, head_act=1, out=p_out)
        predictions["pose_enc"] = pose_list[-1]
        predictions["pose_enc_list"] = pose_list
        predictions["depth"] = d_out[0].view(B, S, H, W, 1)
        predictions["depth_conf"] = d_out[1].view(B, S, H, W)
        predictions["world_points"] = p_out[0].view(B, S, H, W, 3)
        predictions["world_points_conf"] = p_out[1].view(B, S, H, W)
        predictions["images"] = images
        return predictions
