"""Parameter containers that reproduce the reference checkpoint schema (1 505 keys for the full model,
SURVEY.md section 8b) so ``load_state_dict(strict=True)`` of a reference checkpoint works unchanged
(reference inference.py:323-324).  These modules own tensors; the four the reference calls on their own (aggregator,
camera_head, depth_head, point_head: ``Component``) have a forward() that runs on the engine of the OmniVGGT owning them.
Shapes follow the reference constructors cited per class."""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn as nn


def _p(*shape) -> nn.Parameter:
    return nn.Parameter(torch.empty(*shape), requires_grad=False)


class WB(nn.Module):
    """weight (+ bias) holder: nn.Linear / nn.LayerNorm / nn.Conv2d / nn.ConvTranspose2d parameters."""

    def __init__(self, wshape: Sequence[int], bias: bool = True, bshape: Sequence[int] = None):
        super().__init__()
        self.weight = _p(*wshape)
        if bias:
            self.bias = _p(*(bshape if bshape is not None else (wshape[0],)))


class Gamma(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.gamma = _p(dim)          # layers/layer_scale.py:26


class AttnParams(nn.Module):
    """layers/attention.py:21-48."""

    def __init__(self, dim, head_dim, qk_norm):
        super().__init__()
        self.qkv = WB((3 * dim, dim))
        if qk_norm:
            self.q_norm = WB((head_dim,))
            self.k_norm = WB((head_dim,))
        self.proj = WB((dim, dim))


class MlpParams(nn.Module):
    """layers/mlp.py:16-32."""

    def __init__(self, dim, hidden, out=None):
        super().__init__()
        self.fc1 = WB((hidden, dim))
        self.fc2 = WB((out or dim, hidden))


class BlockParams(nn.Module):
    """layers/block.py:27-79."""

    def __init__(self, dim, heads, qk_norm, mlp_ratio=4, layerscale=True):
        super().__init__()
        self.norm1 = WB((dim,))
        self.attn = AttnParams(dim, dim // heads, qk_norm)
        if layerscale:
            self.ls1 = Gamma(dim)
        self.norm2 = WB((dim,))
        self.mlp = MlpParams(dim, int(dim * mlp_ratio))
        if layerscale:
            self.ls2 = Gamma(dim)


class PatchEmbedParams(nn.Module):
    """layers/patch_embed.py:65: Conv2d(in_chans, embed_dim, k = s = patch)."""

    def __init__(self, in_chans, dim, patch):
        super().__init__()
        self.proj = WB((dim, in_chans, patch, patch))


class DinoParams(nn.Module):
    """layers/vision_transformer.py:94-153 (DINOv2 ViT with registers, LayerScale, no mask token)."""

    def __init__(self, img_size, patch, dim, depth, heads, num_register_tokens):
        super().__init__()
        self.patch_embed = PatchEmbedParams(3, dim, patch)
        self.cls_token = _p(1, 1, dim)
        self.pos_embed = _p(1, (img_size // patch) ** 2 + 1, dim)
        self.register_tokens = _p(1, num_register_tokens, dim)
        self.blocks = nn.ModuleList([BlockParams(dim, heads, qk_norm=False) for _ in range(depth)])
        self.norm = WB((dim,))
        self.heads = heads


class Component(nn.Module):
    """A submodule with the reference's call signature.  Its forward delegates to the OmniVGGT that owns it, held as a weak
    reference in ``_owner`` (set by OmniVGGT.__setattr__ with object.__setattr__: not a parameter, buffer or child module, so
    parameters(), state_dict() and _modules are those of a plain container)."""

    def owner(self):
        ref = self.__dict__.get("_owner")
        m = ref() if ref is not None else None
        if m is None or not any(m._modules.get(n) is self for n in ("aggregator", "camera_head", "depth_head", "point_head")):
            raise RuntimeError(f"{type(self).__name__} is called through the OmniVGGT it belongs to; this one is not attached to one")
        return m

    def __getstate__(self):            # weak references do not pickle; OmniVGGT.__setstate__ sets the copy's
        state = dict(super().__getstate__())
        state.pop("_owner", None)
        return state


class AggregatorParams(Component):
    """models/aggregator.py:52-148 + models/omnivggt_aggregator.py:19-80."""

    def __init__(self, img_size, patch, dim, depth, head_dim, num_register_tokens, patch_embed, dino_depth, dino_heads):
        super().__init__()
        if patch_embed == "conv":
            self.patch_embed = PatchEmbedParams(3, dim, patch)
        else:
            self.patch_embed = DinoParams(img_size, patch, dim, dino_depth, dino_heads, num_register_tokens)
        heads = dim // head_dim
        self.frame_blocks = nn.ModuleList([BlockParams(dim, heads, qk_norm=True) for _ in range(depth)])
        self.global_blocks = nn.ModuleList([BlockParams(dim, heads, qk_norm=True) for _ in range(depth)])
        self.camera_token = _p(1, 2, 1, dim)
        self.register_token = _p(1, 2, num_register_tokens, dim)
        self.depth_placeholder = _p(1, 1, dim)
        self.pose_embeddings = nn.ModuleList([WB((dim, 9)) for _ in range(depth + 1)])
        self.camera_adapters = nn.ModuleList([WB((dim, dim)) for _ in range(depth + 1)])
        self.depth_patch_embed = PatchEmbedParams(2, dim, patch)

    def forward(self, images, extrinsics=None, intrinsics=None, depth=None, mask=None, depth_gt_index=None, camera_gt_index=None):
        """ZeroAggregator.forward (omnivggt_aggregator.py:130-256) -> (list of depth fp32 [B, S, T, 2C], patch_start_idx)."""
        return self.owner()._call_aggregator(images, extrinsics, intrinsics, depth, mask, depth_gt_index, camera_gt_index)


class RCUParams(nn.Module):
    """heads/dpt_head.py:357-377."""

    def __init__(self, f):
        super().__init__()
        self.conv1 = WB((f, f, 3, 3))
        self.conv2 = WB((f, f, 3, 3))


class FusionParams(nn.Module):
    """heads/dpt_head.py:402-443."""

    def __init__(self, f, has_residual=True):
        super().__init__()
        self.out_conv = WB((f, f, 1, 1))
        if has_residual:
            self.resConfUnit1 = RCUParams(f)
        self.resConfUnit2 = RCUParams(f)


class ScratchParams(nn.Module):
    """heads/dpt_head.py:98-126,:326-354."""

    def __init__(self, out_channels, f, output_dim):
        super().__init__()
        for i, oc in enumerate(out_channels):
            setattr(self, f"layer{i + 1}_rn", WB((f, oc, 3, 3), bias=False))
        self.refinenet1 = FusionParams(f)
        self.refinenet2 = FusionParams(f)
        self.refinenet3 = FusionParams(f)
        self.refinenet4 = FusionParams(f, has_residual=False)
        self.output_conv1 = WB((f // 2, f, 3, 3))
        self.output_conv2 = nn.ModuleDict({"0": WB((32, f // 2, 3, 3)), "2": WB((output_dim, 32, 1, 1))})


class DPTParams(Component):
    """heads/dpt_head.py:43-126."""

    def __init__(self, dim_in, output_dim, features, out_channels):
        super().__init__()
        oc = out_channels
        self.norm = WB((dim_in,))
        self.projects = nn.ModuleList([WB((c, dim_in, 1, 1)) for c in oc])
        self.resize_layers = nn.ModuleDict({
            "0": WB((oc[0], oc[0], 4, 4), bshape=(oc[0],)),     # ConvTranspose2d k4 s4 (weight [Cin,Cout,k,k])
            "1": WB((oc[1], oc[1], 2, 2), bshape=(oc[1],)),     # ConvTranspose2d k2 s2
            "3": WB((oc[3], oc[3], 3, 3)),                      # Conv2d k3 s2 p1
        })
        self.scratch = ScratchParams(oc, features, output_dim)
        self.output_dim = output_dim

    def forward(self, aggregated_tokens_list, images, patch_start_idx, frames_chunk_size=8):
        """DPTHead.forward (dpt_head.py:128-183) -> (preds [B, S, H, W, output_dim - 1], conf [B, S, H, W])."""
        return self.owner()._call_dpt(self, aggregated_tokens_list, images, patch_start_idx, frames_chunk_size)


class CameraHeadParams(Component):
    """heads/camera_head.py:26-81."""

    def __init__(self, dim_in, trunk_depth, heads):
        super().__init__()
        self.trunk = nn.ModuleList([BlockParams(dim_in, heads, qk_norm=False) for _ in range(trunk_depth)])
        self.token_norm = WB((dim_in,))
        self.trunk_norm = WB((dim_in,))
        self.empty_pose_tokens = _p(1, 1, 9)
        self.embed_pose = WB((dim_in, 9))
        self.poseLN_modulation = nn.ModuleDict({"1": WB((3 * dim_in, dim_in))})
        self.pose_branch = MlpParams(dim_in, dim_in // 2, out=9)
        self.heads = heads

    def forward(self, aggregated_tokens_list, num_iterations=4):
        """CameraHead.forward (camera_head.py:83-103) -> list of num_iterations pose encodings [B, S, 9]."""
        return self.owner()._call_camera(aggregated_tokens_list, num_iterations)


@torch.no_grad()
def init_parameters(module: nn.Module, seed: int = 0, dezero: bool = False) -> None:
    """Random init on the parameters' device.  dezero=False mimics the reference's construction-time statistics
    (zero camera adapters omnivggt_aggregator.py:70-72, LayerScale 0.01, 1e-6 special tokens aggregator.py:136-137);
    dezero=True gives every tensor an O(1) role (used for synthetic-weight parity tests and benchmarks)."""
    dev = next(module.parameters()).device
    g = torch.Generator(device=dev).manual_seed(seed)
    for name, p in module.named_parameters():
        leaf = name.rsplit(".", 1)[-1]
        shape = p.shape
        mean, std = 0.0, 0.02
        if leaf == "gamma":
            mean, std = (0.25, 0.05) if dezero else ((1.0, 0.0) if ".patch_embed." in name else (0.01, 0.0))
        elif "norm" in name and leaf == "weight" and p.dim() == 1:
            mean, std = 1.0, (0.1 if dezero else 0.0)
        elif leaf == "bias":
            std = 0.05 if dezero else 0.0
        elif leaf in ("camera_token", "register_token", "cls_token", "register_tokens"):
            std = 0.5 if dezero else 1e-6
        elif leaf in ("depth_placeholder", "empty_pose_tokens"):
            std = 0.3 if dezero else 0.0
        elif leaf == "pos_embed":
            std = 0.2 if dezero else 0.02
        elif leaf == "weight" and p.dim() >= 2:
            if "camera_adapters" in name and not dezero:
                std = 0.0
            else:
                fan_in = shape[0] if ("resize_layers.0" in name or "resize_layers.1" in name) else int(p[0].numel())
                std = fan_in ** -0.5
        if std == 0.0:
            p.fill_(mean)
        else:
            p.copy_(torch.randn(shape, generator=g, device=dev) * std + mean)
