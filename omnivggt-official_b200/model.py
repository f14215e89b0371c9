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

import numpy as np
import torch
import torch.nn as nn

try:  # keep from_pretrained / save_pretrained like the reference (omnivggt.py:3,:10)
    from huggingface_hub import PyTorchModelHubMixin
except Exception:  # pragma: no cover
    class PyTorchModelHubMixin:  # type: ignore
        pass

from . import torch_parts as TP
from .params import AggregatorParams, CameraHeadParams, Component, DPTParams, init_parameters

_RESNET_MEAN = (0.485, 0.456, 0.406)   # reference models/aggregator.py:22-23
_RESNET_STD = (0.229, 0.224, 0.225)
_HEADS = ("camera_head", "depth_head", "point_head")
_DPT_HEADS = (("depth_head", 0), ("point_head", 1))          # name, head_act (exp / inverse-log)


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
        impl = self._forward_cp if self._cp is not None else self._forward_impl
        if self.use_cuda_graph and images.is_cuda and not torch.cuda.is_current_stream_capturing():
            return self._forward_graphed(eng, impl, *args)
        return impl(eng, *args)

    def _check_inputs(self, images, extrinsics, intrinsics, depth, mask, depth_gt_index, camera_gt_index):
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
        return images, depth_idx, cam_idx

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
        heads = self._dpt_heads()
        slots, cam_loc = eng.aggregate(patch, inj, depth, mask, depth_idx, 1, n, H, W, set(self.dpt_layers), cp=cp, views_total=S,
                                       slots=bool(heads))
        out: Dict[str, object] = {}
        if self.camera_head is not None:   # [S, 2C] gathered by peer stores: the camera head attends across all views
            pose_list = self._camera(eng, cp.cam_all, 1, S)
            out["pose_enc"], out["pose_enc_list"] = pose_list[-1], pose_list
        eng.warm_tables(H, W)
        for name, act in heads:
            preds, conf = eng.dpt(name, slots, self.dpt_layers, n, H, W, head_act=act)
            self._put_dpt(out, name, preds, conf, 1, n, H, W)
        out["images"], out["view_range"] = images[:, sl], (v0, v0 + n)
        return out

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
        forward(); the layers are written by the snapshot pass of the aggregator (ovg_aggregator_forward_layers)."""
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
    def _check_views(predictions: Dict[str, object], source: str, conf_percent: float, conf_floor: float,
                     frame: Optional[int], scene: int, mask_sky) -> int:
        """The argument checks of point_cloud, mesh and matches, before any library call; returns the scene's view count."""
        if source not in ("depth", "pointmap"):
            raise ValueError(f"source must be 'depth' or 'pointmap', got {source!r}")
        if not 0.0 <= conf_percent <= 100.0:
            raise ValueError("conf_percent must be in [0, 100]")
        if conf_floor < 0.0:
            raise ValueError("conf_floor must be >= 0")        # the reference's floors are 1e-5 and 0.1
        OmniVGGT._check_mask_sky(mask_sky, predictions, scene)
        images = predictions["images"]
        S = (images[scene] if images.dim() == 5 else images).shape[0]
        if frame is not None and not 0 <= frame < S:
            raise IndexError(f"frame {frame} out of range for {S} views")
        return S

    @staticmethod
    def _kept_views(predictions: Dict[str, object], source: str, conf_percent: float, conf_floor: float,
                    frame: Optional[int], scene: int, mask_sky):
        """The views point_cloud, mesh and matches work on and their keep mask, after _check_views: the scene's source, its
        confidence times non-sky over all views, then the frame, then conf >= percentile(conf, conf_percent) and
        conf > conf_floor.  Returns (images fp32 [F,3,H,W], extrinsic [S,3,4], points fp32 [F,H,W,3], mask uint8 [F,H,W],
        threshold 0-d, first view f0), the images, points and mask contiguous."""
        from . import ops
        images, ext, points, conf = OmniVGGT._scene_source(predictions, source, scene)
        conf = OmniVGGT._sky_conf(mask_sky, images, conf, scene)
        f0 = 0 if frame is None else frame
        if frame is not None:
            images, points, conf = images[frame:frame + 1], points[frame:frame + 1], conf[frame:frame + 1]
        mask, thr, _ = ops.conf_percentile_mask(conf.float().contiguous(), conf_percent, conf_floor)
        if conf_percent == 0.0:
            thr = torch.zeros((), device=images.device, dtype=torch.float32)   # same mask: conf > conf_floor >= 0 implies conf >= 0
        return images.contiguous(), ext, points.float().contiguous(), mask, thr, f0

    @staticmethod
    def _scene_source(predictions: Dict[str, object], source: str, scene: int):
        """(images fp32 [S,3,H,W], extrinsic [S,3,4], points [S,H,W,3], conf [S,H,W]) of one scene.  ``source="depth"``:
        ``world_points_from_depth`` (unprojected here when ``postprocess`` has not run) with ``depth_conf``; ``"pointmap"``:
        ``world_points`` with ``world_points_conf``."""
        from . import ops

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
        return images, ext, points, conf

    @staticmethod
    def _segment_views(images: torch.Tensor, conf: Optional[torch.Tensor] = None):
        """ops.segment_sky over the views of images fp32 [S,3,H,W], read in place when each channel plane is contiguous."""
        from . import ops
        S, _, H, W = images.shape
        if images.stride(3) != 1 or images.stride(2) != W:
            images = images.contiguous()
        return ops.segment_sky(images, S, H, W, images.stride(0), 1, images.stride(1), conf)

    @staticmethod
    @torch.no_grad()
    def sky_mask(predictions: Dict[str, object], *, scene: int = 0) -> torch.Tensor:
        """The sky of every view of one scene: the reference's model-free segment_sky (viz.py:357-393) on the images the model
        saw, ``predictions["images"]`` fp32 [S,3,H,W] (or [B,S,3,H,W]), all views in one call with no host read.  Returns bool
        [S, H, W] on the device, True = sky; ``point_cloud``, ``mesh`` and ``matches`` take it as ``mask_sky``."""
        images = predictions["images"]
        images = (images[scene] if images.dim() == 5 else images).float()
        sky, _ = OmniVGGT._segment_views(images)
        return sky.bool()

    @staticmethod
    def _check_mask_sky(mask_sky, predictions: Dict[str, object], scene: int) -> None:
        """mask_sky is a bool, or a bool tensor [S, H, W] / [B, S, H, W] (True = sky) on the images' device."""
        if isinstance(mask_sky, (bool, np.bool_)):
            return
        if not torch.is_tensor(mask_sky) or mask_sky.dtype != torch.bool:
            raise ValueError(f"mask_sky must be a bool or a bool tensor, got {getattr(mask_sky, 'dtype', type(mask_sky))}")
        images = predictions["images"]
        want = (tuple(images.shape[:2]) if images.dim() == 5 else (images.shape[0],)) + tuple(images.shape[-2:])
        if mask_sky.dim() == 4 and images.dim() == 5:
            ok = tuple(mask_sky.shape) == want
        else:
            ok = tuple(mask_sky.shape) == want[-3:]
        if not ok:
            raise ValueError(f"mask_sky must have shape [S, H, W] = {list(want[-3:])}"
                             + (f" or [B, S, H, W] = {list(want)}" if images.dim() == 5 else "") + f", got {list(mask_sky.shape)}")
        if mask_sky.device != images.device:
            raise ValueError(f"mask_sky is on {mask_sky.device}, the images on {images.device}")

    @staticmethod
    def _sky_conf(mask_sky, images: torch.Tensor, conf: torch.Tensor, scene: int) -> torch.Tensor:
        """conf [S,H,W] of the scene times non-sky, over all S views, as visual_util.py:186-188 does before the frame selection
        and the percentile.  mask_sky False: conf unchanged, no launch."""
        from . import ops
        if isinstance(mask_sky, (bool, np.bool_)):
            if not mask_sky:
                return conf
            _, out = OmniVGGT._segment_views(images, conf.float().contiguous())
            return out
        sky = mask_sky[scene] if mask_sky.dim() == 4 else mask_sky
        return ops.sky_mask_conf(conf.float().contiguous(), sky.contiguous().view(torch.uint8))

    @staticmethod
    @torch.no_grad()
    def matches(predictions: Dict[str, object], pairs=None, *, source: str = "depth", conf_percent: float = 50.0,
                conf_floor: float = 1e-5, scene: int = 0, mask_sky=False) -> List[Dict[str, object]]:
        """Dense cross-view correspondences of one scene by reciprocal nearest neighbours of the predicted points (the
        DUSt3R-family recipe on utils/geometry.py:435-451 find_reciprocal_matches and :15-37 xy_grid), on the device.

        ``source`` and the keep mask are ``point_cloud``'s: conf >= percentile(conf over the scene's S views, conf_percent) and
        conf > conf_floor.  For each pair (i, j) (default: every i < j), P1 and P2 are the kept points of views i and j in
        row-major order, and the result is ``{"xy_i", "xy_j", "count"}`` with ``xy_j = grid_j[kept_j][reciprocal_in_P2]`` and
        ``xy_i = grid_i[kept_i][nn2_in_P1][reciprocal_in_P2]``: int64 [count, 2] (x, y) pixel coordinates on the device.
        Every view's index is built once; all pairs are queried in one pass; the match counts are the one host read.  Kept
        points that are not finite raise ValueError; a view with no kept point has no matches.  ``mask_sky``: as in
        ``point_cloud``."""
        from . import geometry, ops
        S = OmniVGGT._check_views(predictions, source, conf_percent, conf_floor, None, scene, mask_sky)
        pair_arr = geometry.check_pairs(pairs, S)
        if len(pair_arr) == 0:
            return []
        images, _, points, mask, _, _ = OmniVGGT._kept_views(predictions, source, conf_percent, conf_floor, None, scene, mask_sky)
        _, _, H, W = images.shape
        mt = ops.Matcher(points.view(S, H * W, 3), mask.view(S, H * W), torch.from_numpy(pair_arr).to(images.device))
        counts, nonfinite = mt.counts()
        if nonfinite:
            raise ValueError("kept points must be finite (cKDTree: data must be finite, check for nan or inf values)")
        xy_i, xy_j = mt.gather(sum(counts), W)
        return [{"xy_i": a, "xy_j": b, "count": c} for a, b, c in zip(xy_i.split(counts), xy_j.split(counts), counts)]

    @staticmethod
    @torch.no_grad()
    def point_cloud(predictions: Dict[str, object], *, source: str = "depth", conf_percent: float = 50.0,
                    conf_floor: float = 1e-5, frame: Optional[int] = None, mask_black_bg: bool = False,
                    mask_white_bg: bool = False, scene: int = 0, mask_sky=False) -> Dict[str, torch.Tensor]:
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
        with E0 the first selected camera (visual_util.py:320-341).  The kept count and E0 are the only device-to-host reads.

        ``mask_sky`` (the reference's --mask_sky, visual_util.py:140-188): False, no sky masking; True, the sky of every view
        by ``sky_mask``; or a bool tensor [S,H,W] / [B,S,H,W], True = sky (a reference mask file m, uint8 255 = non-sky, at
        H x W is ``m == 0``).  The confidence of every view becomes conf * non-sky before the frame selection and the
        percentile, as the reference orders it; no host read is added."""
        from . import ops
        OmniVGGT._check_views(predictions, source, conf_percent, conf_floor, frame, scene, mask_sky)
        images, ext, points, mask, thr, f0 = OmniVGGT._kept_views(predictions, source, conf_percent, conf_floor, frame, scene,
                                                                  mask_sky)
        F, _, H, W = images.shape
        dev = images.device
        ws = ops.point_cloud_workspace(F * H * W, dev)
        cnt = ops.point_cloud_count(mask, images, ws, mask_black_bg, mask_white_bg)
        center = ops.point_cloud_center(points, ws)
        host = ops.host_read(torch.cat([cnt.double().reshape(1), ext[f0].double().reshape(-1)]))   # count < 2^31: exact
        n = int(host[0])
        align = OmniVGGT._align(host[1:].view(3, 4)).to(dev)
        if n == 0:
            return {"points": torch.empty(0, 3, device=dev), "colors": torch.empty(0, 3, device=dev, dtype=torch.uint8),
                    "frame": torch.empty(0, device=dev, dtype=torch.int32), "conf_threshold": thr, "center": center,
                    "scale": torch.ones((), device=dev), "align": align}
        pts, cols, fr, xyz = ops.point_cloud_gather(points, mask, images, ws, n, mask_black_bg, mask_white_bg, f0)
        scale = ops.point_cloud_scale(xyz, n, ws)
        return {"points": pts, "colors": cols, "frame": fr, "conf_threshold": thr, "center": center, "scale": scale,
                "align": align}

    @staticmethod
    def _align(e0: torch.Tensor) -> torch.Tensor:
        """inv(E0) diag(1,-1,-1,1) R_y(180), fp64 [4,4] on the host, from the host camera E0 [3,4] (visual_util.py:320-341)."""
        e = torch.eye(4, dtype=torch.float64)
        e[:3, :4] = e0
        gl = torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0], dtype=torch.float64))
        rot_y = torch.diag(torch.tensor([-1.0, 1.0, -1.0, 1.0], dtype=torch.float64))
        return torch.linalg.inv(e) @ gl @ rot_y

    @staticmethod
    @torch.no_grad()
    def mesh(predictions: Dict[str, object], *, source: str = "depth", conf_percent: float = 50.0, conf_floor: float = 1e-5,
             frame: Optional[int] = None, mask_black_bg: bool = False, mask_white_bg: bool = False, scene: int = 0,
             layout: str = "reference", mask_sky=False) -> Dict[str, torch.Tensor]:
        """The coloured triangle mesh of one scene's point maps, built on the device (libovg kernels): the DUSt3R-family
        recipe of viz.py:40-89, ``cat_meshes([pts3d_to_trimesh(colors[f], points[f], keep[f]) for f in views])``.

        ``source``, ``conf_percent``, ``conf_floor``, ``frame``, the background masks and ``scene`` select the views and the
        kept pixels exactly as in ``point_cloud``; colours are (images * 255).astype(uint8).  Every pixel quad gives two
        triangles, (tl, tr, bl) and (tr, bl, br); a triangle is kept when its three pixels are.

        ``layout="reference"``: ``vertices`` fp32 [F*H*W, 3] (every point of the selected views), ``face_colors`` uint8 [n, 3]
        and ``faces`` int64 [n, 3], as viz.py returns them: per view the kept (tl, tr, bl) triangles, the same reversed, the kept
        (tr, bl, br) triangles, the same reversed, each in row-major order; colours from tl and br.
        ``layout="glb"``: ``positions`` fp32 [m, 3] and ``colors`` uint8 [m, 3] of the vertices the forward triangles use, in
        index order, each with its own pixel's colour, and ``indices`` int32 [k, 3] of the forward triangles only, for
        ``glb.write_mesh_glb`` (whose material is double-sided in place of the reversed copies).
        Both add ``conf_threshold`` and ``align``, as ``point_cloud`` returns them.  The three totals and the first camera are
        read back together: the one host synchronisation.  ``mask_sky``: as in ``point_cloud``."""
        from . import ops
        OmniVGGT._check_views(predictions, source, conf_percent, conf_floor, frame, scene, mask_sky)
        if layout not in ("reference", "glb"):
            raise ValueError(f"layout must be 'reference' or 'glb', got {layout!r}")
        images, ext, points, mask, thr, f0 = OmniVGGT._kept_views(predictions, source, conf_percent, conf_floor, frame, scene,
                                                                  mask_sky)
        F, _, H, W = images.shape
        mesher = ops.Mesher(mask.view(-1), images, F, H, W, mask_black_bg, mask_white_bg)
        host = ops.host_read(torch.cat([mesher.totals.double(), ext[f0].double().reshape(-1)]))   # totals < 2^33: exact
        n_ref, n_used, n_fwd = (int(v) for v in host[:3].tolist())
        align = OmniVGGT._align(host[3:].view(3, 4)).to(images.device)
        if layout == "glb":
            pos, cols, idx = mesher.compact(points.view(-1, 3), n_used, n_fwd)
            return {"positions": pos, "colors": cols, "indices": idx, "conf_threshold": thr, "align": align}
        faces, face_colors = mesher.faces(n_ref)
        return {"vertices": points.view(-1, 3).clone(), "face_colors": face_colors, "faces": faces, "conf_threshold": thr,
                "align": align}

    # ---------------------------------------------------------------------------------------------- CUDA graph replay
    def _forward_graphed(self, eng, impl, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx):
        """Same computation, launched from a captured CUDA graph (a forward is >1000 kernel launches; issuing them from
        Python costs about as much host time as the GPU needs to run them).  A graph is captured the third time a
        (shape, index-list) signature is seen; inputs are copied into static buffers, outputs are cloned."""
        need_c, need_d = len(cam_idx) > 0, len(depth_idx) > 0
        def sig(t):
            return None if t is None else (tuple(t.shape), t.dtype)
        heads = tuple(getattr(self, n) is not None for n in _HEADS)
        key = (impl.__name__, sig(images), tuple(depth_idx), tuple(cam_idx), sig(extrinsics) if need_c else None,
               sig(intrinsics) if need_c else None, sig(depth) if need_d else None, sig(mask) if need_d else None, heads)
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
        if "pose_enc_list" in out:
            res["pose_enc_list"] = [t.clone() for t in out["pose_enc_list"]]
            res["pose_enc"] = res["pose_enc_list"][-1]
        res["images"] = images if "view_range" not in out else images[:, out["view_range"][0]:out["view_range"][1]]
        return res

    def _camera(self, eng, cam_tokens, B, S):
        if eng.h_cam is not None:
            return eng.camera_head(cam_tokens, B, S)
        return TP.camera_head(self.camera_head, cam_tokens.view(B, S, -1), dtype=self.camera_dtype)

    def _aggregate(self, eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx, slots=True, layers=None):
        """Patchifier, camera / depth injection and the aggregator: (bf16 slots of the kept layers, fp32 camera tokens [K, 2C])."""
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
        return eng.aggregate(patch, inj, depth, mask, depth_idx, B, S, H, W, keep, slots=slots, layers=layers)

    def _forward_impl(self, eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx):
        B, S, Cin, H, W = images.shape
        K = B * S
        heads = self._dpt_heads()                 # the heads set to None are skipped, as the reference does (omnivggt.py:46-62)
        cam_on = self.camera_head is not None
        slots, cam_tokens = self._aggregate(eng, images, extrinsics, intrinsics, depth, mask, depth_idx, cam_idx, slots=bool(heads))

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
        if main is not None and self.head_streams and cam_on + len(heads) > 1:
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
            self._put_dpt(predictions, name, *outs[name], B, S, H, W)
        predictions["images"] = images
        return predictions
