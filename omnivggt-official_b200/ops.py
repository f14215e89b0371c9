"""Thin tensor-level wrappers over the libovg C ABI (device pointers + current stream).  Pure plumbing:
argument checking and pointer extraction; every byte of arithmetic happens in the CUDA library."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

from . import _lib as L

BF16 = torch.bfloat16
F32 = torch.float32


def _on_device(t: torch.Tensor) -> bool:
    return t.is_cuda


def check_operand(t: torch.Tensor, name: str, dtype, *, shape=None, numel: Optional[int] = None, contiguous: bool = False,
                  unit_stride: bool = False) -> None:
    """The contract of an operand whose pointer goes to libovg, which cannot check it.  TypeError unless it is on the device
    with ``dtype`` (a tuple: any of them; None: any); ValueError unless it has ``shape`` (None: any size there) and ``numel``
    elements and, where asked, is contiguous / has a unit stride in the last dim."""
    dtypes = dtype if isinstance(dtype, tuple) else (dtype,)
    if (dtype is not None and t.dtype not in dtypes) or not _on_device(t):
        want = "tensor" if dtype is None else " or ".join(map(str, dtypes))
        raise TypeError(f"{name}: expected cuda {want}, got {t.device} {t.dtype}")
    if shape is not None and (t.dim() != len(shape) or any(n is not None and n != m for n, m in zip(shape, t.shape))):
        want = ", ".join("*" if n is None else str(n) for n in shape)
        raise ValueError(f"{name}: expected shape [{want}], got {list(t.shape)}")
    if numel is not None and t.numel() != numel:
        raise ValueError(f"{name}: expected {numel} elements, got {t.numel()} (shape {list(t.shape)})")
    if contiguous and not t.is_contiguous():
        raise ValueError(f"{name}: expected a contiguous tensor, got shape {list(t.shape)} with strides {t.stride()}")
    if unit_stride and t.stride(-1) != 1:
        raise ValueError(f"{name}: expected a unit stride in the last dim, got strides {t.stride()}")


def workspace_bytes(query: str, *args) -> int:
    """libovg's size query ``query`` (ovg_*_workspace_bytes / *_scratch_bytes) for args; OvgError if it rejects them (< 0)."""
    n = getattr(L.lib(), query)(*args)
    if n < 0:
        raise L.OvgError(f"libovg: {query} rejected its arguments (returned {n})")
    return n


def workspace(device, query: str, *args) -> torch.Tensor:
    """uint8 workspace of workspace_bytes(query, *args) bytes on ``device``."""
    return torch.empty(workspace_bytes(query, *args), device=device, dtype=torch.uint8)


def gemm(a: torch.Tensor, b: torch.Tensor, *, m: Optional[int] = None, taps: Optional[Sequence[int]] = None,
         epi: int = L.EPI_BF16, block_n: int = 0, **kw) -> None:
    """a: bf16 [rows, a_cols] (last dim contiguous), b: bf16 [n, taps*a_cols] -- or both fp16 (EPI_BF16 / EPI_HEADTAIL only:
    skips and the output are then fp16 too).  kw: fields of ovg_gemm_args."""
    f16 = a.dtype == torch.float16
    if f16:
        if epi not in (L.EPI_BF16, L.EPI_HEADTAIL):
            raise ValueError(f"fp16 operands: EPI_BF16 / EPI_HEADTAIL only, got epi {epi}")
        kw = dict(kw, f16=1)
    taps = list(taps) if taps is not None else [0]
    check_operand(a, "a", torch.float16 if f16 else BF16, shape=(None, None), unit_stride=True)
    check_operand(b, "b", a.dtype, shape=(None, a.shape[1] * len(taps)), unit_stride=True)
    g = L.GemmArgs()
    g.a, g.a_rows, g.a_cols, g.lda = a.data_ptr(), a.shape[0], a.shape[1], a.stride(0)
    g.b, g.n, g.ldb = b.data_ptr(), b.shape[0], b.stride(0)
    g.m = a.shape[0] if m is None else m
    g.num_taps = len(taps)
    for i, t in enumerate(taps):
        g.tap_off[i] = int(t)
    g.epi = epi
    g.block_n = block_n
    keep = []
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            check_operand(v, k, None, contiguous=True)
            keep.append(v)
            setattr(g, k, v.data_ptr())
        elif v is not None:
            setattr(g, k, v)
    L.check(L.lib().ovg_gemm(g, L.stream()))


def linear_bf16(a, w, bias=None, act=L.ACT_NONE, out=None, block_n=0):
    out = out if out is not None else torch.empty(a.shape[0], w.shape[0], device=a.device, dtype=BF16)
    gemm(a, w, epi=L.EPI_BF16, bias=bias, act=act, out=out, ldo=out.stride(0), block_n=block_n)
    return out


def linear_resid(a, w, bias, gamma, x, row_index=None, block_n=0):
    """x(fp32)[row] += gamma * (a @ w^T + bias)."""
    check_operand(x, "x", F32)
    gemm(a, w, epi=L.EPI_RESID, bias=bias, gamma=gamma, out=x, ldo=x.stride(0), row_index=row_index, block_n=block_n)
    return x


def rope_tables(maxpos: int, device, base: float = 100.0):
    """fp32 cos/sin [maxpos, 16] exactly as the reference builds them (layers/rope.py:103-114, head half = 32)."""
    exponents = torch.arange(0, 32, 2, device=device).float() / 32
    inv_freq = 1.0 / (base ** exponents)
    ang = torch.arange(maxpos, device=device, dtype=inv_freq.dtype)[:, None] * inv_freq[None]
    return ang.cos().contiguous(), ang.sin().contiguous()


def qkv_proj(a, w, bias, qn_w, qn_b, kn_w, kn_b, q, k, v, *, ntok, T, nspecial=0, wp=1, rope_cos=None, rope_sin=None,
             block_n=0):
    """QKV linear with fused epilogue.  q/k LayerNorm when qn_w is given, 2-D RoPE when rope tables are given."""
    C = w.shape[1]
    gemm(a, w, epi=L.EPI_QKV, bias=bias, q_out=q, k_out=k, v_out=v, C=C, ntok=ntok, T=T, nspecial=nspecial, wp=wp,
         maxpos=0 if rope_cos is None else rope_cos.shape[0], qn_w=qn_w, qn_b=qn_b, kn_w=kn_w, kn_b=kn_b,
         rope_cos=rope_cos, rope_sin=rope_sin, qk_norm=int(qn_w is not None), rope=int(rope_cos is not None),
         qscale=(1.0 / math.sqrt(64.0)) * math.log2(math.e), block_n=block_n)


def attention(q, k, v, out, batch: int, heads: int, nq: int, nkv: Optional[int] = None, scratch=None):
    """q [batch, heads, nq, 64] against k, v [batch, heads, nkv, 64] (nkv defaults to nq) -> out [batch, nq, heads*64].
    scratch: uint8 buffer of ovg_attention_scratch_bytes() -> long sequences may split the tiles of the last CTA wave over the keys."""
    for t, name in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        check_operand(t, name, BF16, contiguous=True)
    L.check(L.lib().ovg_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), batch, heads, nq,
                                  nq if nkv is None else nkv, L.ptr(scratch), 0 if scratch is None else scratch.numel(),
                                  L.stream()))
    return out


def attention_scratch(device):
    return workspace(device, "ovg_attention_scratch_bytes")


def layernorm(x, out, w=None, b=None, eps=1e-5, rows=None, grp_out=0, grp_in=0, grp_off=0):
    check_operand(x, "x", (F32, BF16), unit_stride=True)
    check_operand(out, "out", (F32, BF16, torch.float16), unit_stride=True)
    x2 = x if x.dim() == 2 else x.reshape(-1, x.shape[-1])
    o2 = out if out.dim() == 2 else out.reshape(-1, out.shape[-1])
    rows = o2.shape[0] if rows is None else rows
    L.check(L.lib().ovg_layernorm(x2.data_ptr(), int(x.dtype == BF16), x2.stride(0), o2.data_ptr(),
                                  {BF16: 0, F32: 1, torch.float16: 2}[out.dtype], o2.stride(0), rows,
                                  o2.shape[1], L.ptr(w), L.ptr(b), eps, grp_out, grp_in, grp_off, L.stream()))
    return out


def assemble_tokens(x, patch, cam_tok, reg_tok, inj0, placeholder, has_depth, K, S, T, R, C, view_base: int = 0):
    L.check(L.lib().ovg_assemble_tokens(x.data_ptr(), patch.data_ptr(), cam_tok.data_ptr(), reg_tok.data_ptr(),
                                        inj0.data_ptr(), placeholder.data_ptr(), has_depth.data_ptr(), K, S, T, R, C,
                                        view_base, L.stream()))


def inject_snapshot(x, inj, slot, cam_out, K, T, C, coff):
    L.check(L.lib().ovg_inject_snapshot(x.data_ptr(), L.ptr(inj), L.ptr(slot), L.ptr(cam_out), K, T, C, coff,
                                        L.stream()))


def depth_im2col(depth, mask, idx, scratch, cols, B, S, Sd, H, W, patch):
    """Normalisation mean and im2col rows over the same Sd views idx."""
    L.check(L.lib().ovg_depth_im2col(depth.data_ptr(), mask.data_ptr(), idx.data_ptr(), Sd, idx.data_ptr(), Sd,
                                     scratch.data_ptr(), cols.data_ptr(), cols.stride(0), B, S, H, W, patch, L.stream()))


def im2col3x3s2(src, dst, F, h, w, C):
    L.check(L.lib().ovg_im2col3x3s2(src.data_ptr(), dst.data_ptr(), F, h, w, C, L.stream()))


def upsample_bilinear(src, dst, tx, ty, F, h, w, H, W, C):
    """tx [W, C/2], ty [H, C/2]: separable UV position embedding (or both None); src / dst both bf16 or both fp16."""
    check_operand(src, "src", (BF16, torch.float16))
    check_operand(dst, "dst", src.dtype)
    L.check(L.lib().ovg_upsample_bilinear(src.data_ptr(), dst.data_ptr(), L.ptr(tx), L.ptr(ty), F, h, w, H, W, C,
                                          int(src.dtype == torch.float16), L.stream()))


def dpt_tail(src, tx, ty, w3x3, bias, w2, b2, head_act: int, F: int, h: int, w: int, H: int, W: int):
    """Fused resize + position embedding + 3x3 conv 128->32 + ReLU + 1x1 + activations (ovg_dpt_tail).  src: zero-bordered
    [F, h+2, w+2, 128] bf16 / fp16; w3x3 [32, 9*128] same dtype.  Returns (preds fp32 [F,H,W,outc-1], conf fp32 [F,H,W])."""
    check_operand(src, "src", (BF16, torch.float16), contiguous=True)
    check_operand(w3x3, "w3x3", src.dtype, contiguous=True)
    outc = w2.shape[0]
    preds = torch.empty(F, H, W, outc - 1, device=src.device, dtype=F32)
    conf = torch.empty(F, H, W, device=src.device, dtype=F32)
    scratch = workspace(src.device, "ovg_dpt_tail_scratch_bytes", H, W)
    L.check(L.lib().ovg_dpt_tail(src.data_ptr(), L.ptr(tx), L.ptr(ty), w3x3.data_ptr(), bias.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                 outc, head_act, preds.data_ptr(), conf.data_ptr(), F, h, w, H, W, int(src.dtype == torch.float16),
                                 scratch.data_ptr(), L.stream()))
    return preds, conf


def pose_decode(pose_enc, H: int, W: int):
    """pose_enc fp32 [..., 9] -> (extrinsic [..., 3, 4], intrinsic [..., 3, 3], cam2world [..., 3, 4]) on the device."""
    check_operand(pose_enc, "pose_enc", F32)
    pe = pose_enc.contiguous()
    lead = pe.shape[:-1]
    K = pe.numel() // 9
    ext = torch.empty(*lead, 3, 4, device=pe.device, dtype=F32)
    intr = torch.empty(*lead, 3, 3, device=pe.device, dtype=F32)
    c2w = torch.empty(*lead, 3, 4, device=pe.device, dtype=F32)
    L.check(L.lib().ovg_pose_decode(pe.data_ptr(), ext.data_ptr(), intr.data_ptr(), c2w.data_ptr(), K, H, W, L.stream()))
    return ext, intr, c2w


def unproject_depth(depth, intrinsic, cam2world, H: int, W: int):
    """depth fp32 [K, H, W], intrinsic fp32 [K, 3, 3], cam2world fp32 [K, 3, 4] -> world points fp32 [K, H, W, 3]."""
    check_operand(depth, "depth", F32)
    d = depth.contiguous()
    K = d.numel() // (H * W)
    intr, c2w = intrinsic.contiguous(), cam2world.contiguous()
    check_operand(intr, "intrinsic", F32, numel=K * 9)
    check_operand(c2w, "cam2world", F32, numel=K * 12)
    world = torch.empty(K, H, W, 3, device=d.device, dtype=F32)
    L.check(L.lib().ovg_unproject_depth(d.data_ptr(), intr.data_ptr(), c2w.data_ptr(), world.data_ptr(), K, H, W, L.stream()))
    return world


def conf_percentile_mask(conf, percent: float, floor: float = 0.1):
    """(mask uint8 like conf, threshold 0-d fp32 tensor, kept-count 0-d int64 tensor); threshold = numpy.percentile(conf, percent)."""
    check_operand(conf, "conf", F32)
    c = conf.contiguous()
    ws = torch.empty(L.PERCENTILE_WORKSPACE_BYTES // 8 + 1, device=c.device, dtype=torch.int64)
    mask = torch.empty(c.shape, device=c.device, dtype=torch.uint8)
    thr = torch.empty((), device=c.device, dtype=F32)
    cnt = torch.empty((), device=c.device, dtype=torch.int64)
    L.check(L.lib().ovg_conf_percentile_mask(c.data_ptr(), c.numel(), float(percent), float(floor), ws.data_ptr(),
                                             mask.data_ptr(), thr.data_ptr(), cnt.data_ptr(), L.stream()))
    return mask, thr, cnt


def point_cloud_workspace(n: int, device):
    """uint8 workspace of ovg_point_cloud_workspace_bytes(n) for a cloud over n pixels (F*H*W)."""
    return workspace(device, "ovg_point_cloud_workspace_bytes", n)


def point_cloud_count(conf_mask, images, ws, mask_black_bg: bool = False, mask_white_bg: bool = False):
    """conf_mask uint8 [F,H,W], images fp32 [F,3,H,W] -> kept-pixel count (0-d int64 device tensor)."""
    check_operand(images, "images", F32, shape=(None, 3, None, None), contiguous=True)
    F, _, H, W = images.shape
    check_operand(conf_mask, "conf_mask", torch.uint8, numel=F * H * W, contiguous=True)
    cnt = torch.zeros((), device=images.device, dtype=torch.int64)
    L.check(L.lib().ovg_point_cloud_count(conf_mask.data_ptr(), images.data_ptr(), F, H, W, int(mask_black_bg), int(mask_white_bg),
                                          ws.data_ptr(), ws.numel(), cnt.data_ptr(), L.stream()))
    return cnt


def point_cloud_gather(points, conf_mask, images, ws, n_kept: int, mask_black_bg: bool = False, mask_white_bg: bool = False,
                       frame0: int = 0):
    """The n_kept pixels that point_cloud_count kept, in (frame, row, column) order: (points fp32 [n,3], colors uint8 [n,3],
    frame int32 [n], xyz fp32 [3, ld] column copy of the points for point_cloud_scale)."""
    check_operand(images, "images", F32, shape=(None, 3, None, None), contiguous=True)
    F, _, H, W = images.shape
    check_operand(conf_mask, "conf_mask", torch.uint8, numel=F * H * W, contiguous=True)
    check_operand(points, "points", F32, numel=F * H * W * 3, contiguous=True)
    dev = images.device
    ld = (n_kept + 3) // 4 * 4
    pts = torch.empty(n_kept, 3, device=dev, dtype=F32)
    cols = torch.empty(n_kept, 3, device=dev, dtype=torch.uint8)
    frame = torch.empty(n_kept, device=dev, dtype=torch.int32)
    xyz = torch.empty(3, ld, device=dev, dtype=F32)
    L.check(L.lib().ovg_point_cloud_gather(points.data_ptr(), conf_mask.data_ptr(), images.data_ptr(), F, H, W, int(mask_black_bg),
                                           int(mask_white_bg), int(frame0), ws.data_ptr(), ws.numel(), pts.data_ptr(),
                                           cols.data_ptr(), frame.data_ptr(), xyz.data_ptr(), ld, L.stream()))
    return pts, cols, frame, xyz


def point_cloud_center(points, ws):
    """Mean of points fp32 [..., 3] -> fp32 [3] (fp64 sums in a fixed order)."""
    check_operand(points, "points", F32, contiguous=True)
    center = torch.empty(3, device=points.device, dtype=F32)
    L.check(L.lib().ovg_point_cloud_center(points.data_ptr(), points.numel() // 3, ws.data_ptr(), ws.numel(), center.data_ptr(),
                                           L.stream()))
    return center


def point_cloud_scale(xyz, n_kept: int, ws):
    """||percentile(p, 95) - percentile(p, 5)|| over the first n_kept columns of xyz [3, ld] -> 0-d fp32 tensor."""
    check_operand(xyz, "xyz", F32)
    scale = torch.empty((), device=xyz.device, dtype=F32)
    L.check(L.lib().ovg_point_cloud_scale(xyz.data_ptr(), n_kept, xyz.shape[1], ws.data_ptr(), ws.numel(), scale.data_ptr(),
                                          L.stream()))
    return scale


def segment_sky(image, F: int, H: int, W: int, view_stride: int, pixel_stride: int, channel_stride: int,
                conf: Optional[torch.Tensor] = None):
    """Sky of F views (ovg_segment_sky): image uint8 or fp32 on the device, element (f, y, x, c) at f view_stride +
    (y W + x) pixel_stride + c channel_stride.  Returns (sky uint8 [F, H, W], conf fp32 [F, H, W] * non-sky or None)."""
    check_operand(image, "image", (torch.uint8, F32))
    dev = image.device
    sky = torch.empty(F, H, W, device=dev, dtype=torch.uint8)
    conf_out = None
    if conf is not None:
        check_operand(conf, "conf", F32, numel=F * H * W, contiguous=True)
        conf_out = torch.empty(F, H, W, device=dev, dtype=F32)
    ws = workspace(dev, "ovg_sky_workspace_bytes", F, H, W)
    L.check(L.lib().ovg_segment_sky(image.data_ptr(), int(image.dtype == torch.uint8), view_stride, pixel_stride,
                                    channel_stride, F, H, W, L.ptr(conf), ws.data_ptr(), ws.numel(), sky.data_ptr(),
                                    L.ptr(conf_out), L.stream()))
    return sky, conf_out


def sky_mask_conf(conf, sky):
    """conf fp32 [n...] * (sky ? 0 : 1) for a one-byte (bool / uint8 / int8) sky mask of the same size (ovg_sky_mask_conf)."""
    check_operand(conf, "conf", F32, contiguous=True)
    check_operand(sky, "sky", (torch.bool, torch.uint8, torch.int8), numel=conf.numel(), contiguous=True)
    out = torch.empty_like(conf)
    L.check(L.lib().ovg_sky_mask_conf(conf.data_ptr(), sky.data_ptr(), conf.numel(), out.data_ptr(), L.stream()))
    return out


def farthest_point_sample(xyz, npoint: int, start: Optional[torch.Tensor], include_ends: bool = False):
    """Farthest point sampling of B batches (ovg_farthest_point_sample): xyz fp32 [B, N, 3] on the device, start int64 [B] on
    the device (the first index of each batch; None only with include_ends), 1 <= npoint <= N.  Returns int64 [B, npoint]
    in selection order: one library call, one kernel launch, no host read."""
    check_operand(xyz, "xyz", F32, shape=(None, None, 3), contiguous=True)
    B, N = xyz.shape[0], xyz.shape[1]
    if start is not None:
        check_operand(start, "start", torch.int64, numel=B, contiguous=True)
    ws = workspace(xyz.device, "ovg_fps_workspace_bytes", B, N)
    inds = torch.empty(B, npoint, device=xyz.device, dtype=torch.int64)
    L.check(L.lib().ovg_farthest_point_sample(xyz.data_ptr(), B, N, npoint, L.ptr(start), int(include_ends), ws.data_ptr(),
                                              ws.numel(), inds.data_ptr(), L.stream()))
    return inds


def compute_ranking(ext: torch.Tensor, lambda_t: float, normalize: bool, out_dtype, k: int):
    """Camera-distance matrix and ranking of N views (ovg_compute_ranking): ext fp32 or fp64 [N, >=3, >=4] on the device (any
    strides), out_dtype torch.float32 or torch.float64, 1 <= k <= N.  Returns (ranking int64 [N, k], dists [N, N] of
    out_dtype): one library call, two kernel launches, no host read."""
    check_operand(ext, "ext", (F32, torch.float64), shape=(None, None, None))
    if ext.shape[1] < 3 or ext.shape[2] < 4:
        raise ValueError(f"ext: expected shape [*, >=3, >=4], got {list(ext.shape)}")
    if out_dtype not in (F32, torch.float64):
        raise ValueError(f"out_dtype: expected torch.float32 or torch.float64, got {out_dtype}")
    N = ext.shape[0]
    out_f64 = int(out_dtype == torch.float64)
    ws = workspace(ext.device, "ovg_ranking_workspace_bytes", N, out_f64)
    ranking = torch.empty(N, k, device=ext.device, dtype=torch.int64)
    dists = torch.empty(N, N, device=ext.device, dtype=out_dtype)
    L.check(L.lib().ovg_compute_ranking(ext.data_ptr(), int(ext.dtype == torch.float64), N, *ext.stride(), float(lambda_t),
                                        int(normalize), out_f64, k, ws.data_ptr(), ws.numel(), ranking.data_ptr(),
                                        dists.data_ptr(), L.stream()))
    return ranking, dists


def sim3_estimate(src: torch.Tensor, dst: torch.Tensor, keep: Optional[torch.Tensor] = None):
    """Umeyama similarity (ovg_sim3_estimate) mapping src onto dst: fp32 [n, 3] contiguous on the device, keep uint8 [n] or
    None.  Returns (sim3 fp64 [4, 4], stats fp64 [4] = kept count, status, RMS residual, c): five launches, no host read."""
    check_operand(src, "src", F32, shape=(None, 3), contiguous=True)
    n = src.shape[0]
    check_operand(dst, "dst", F32, shape=(n, 3), contiguous=True)
    if keep is not None:
        check_operand(keep, "keep", torch.uint8, numel=n, contiguous=True)
    ws = workspace(src.device, "ovg_sim3_workspace_bytes", n)
    sim3 = torch.empty(4, 4, device=src.device, dtype=torch.float64)
    stats = torch.empty(4, device=src.device, dtype=torch.float64)
    L.check(L.lib().ovg_sim3_estimate(src.data_ptr(), dst.data_ptr(), L.ptr(keep), n, ws.data_ptr(), ws.numel(), sim3.data_ptr(),
                                      stats.data_ptr(), L.stream()))
    return sim3, stats


def sim3_apply(sim3: torch.Tensor, views: int, hw: int, points=(), depth=None, ext=None) -> None:
    """ovg_sim3_apply: points = up to two (in, out) pairs of fp32 [views * hw, 3], depth = (in, out) fp32 [views * hw],
    ext = (in, out) fp32 [views, 3, 4] world-to-camera; every tensor contiguous on the device, the outputs typically slices of
    merged tensors.  sim3 fp64 [4, 4] on the device.  One launch."""
    check_operand(sim3, "sim3", torch.float64, shape=(4, 4), contiguous=True)
    if len(points) > 2:
        raise ValueError(f"points: expected at most two (in, out) pairs, got {len(points)}")
    pairs = list(points) + [None] * (2 - len(points))
    sizes = [views * hw * 3] * 2 + [views * hw, views * 12]
    flat = []
    for name, pair, size in zip(("points[0]", "points[1]", "depth", "ext"), pairs + [depth, ext], sizes):
        if pair is None:
            flat += [None, None]
            continue
        for t in pair:
            check_operand(t, name, F32, numel=size, contiguous=True)
        flat += [pair[0].data_ptr(), pair[1].data_ptr()]
    L.check(L.lib().ovg_sim3_apply(sim3.data_ptr(), views, hw, *flat, L.stream()))


BA_LOSSES = ("trivial", "cauchy")                 # OVG_BA_LOSS_TRIVIAL, OVG_BA_LOSS_CAUCHY


def bundle_adjust(points, offsets, view, observations, extrinsic, intrinsic, *, iterations: int, refine_focal: bool,
                  loss: str, loss_scale: float, trace: bool = False):
    """ovg_bundle_adjust: points fp64 [n, 3], offsets int64 [n + 1], view int32 [m], observations fp64 [m, 2] (COLMAP pixel
    frame), extrinsic fp32 [V, 3, 4], intrinsic fp32 [V, 3, 3], contiguous on one device.  Returns (points fp64 [n, 3],
    extrinsic fp64 [V, 3, 4], intrinsic fp64 [V, 3, 3], error fp64 [n], cost fp64 [2], stats int64 [4] = steps, accepted,
    PCG iterations, status, and with ``trace`` the cost after each step fp64 [iterations], NaN after the last).  No host read."""
    n, m, V = points.shape[0], view.shape[0], extrinsic.shape[0]
    check_operand(points, "points", torch.float64, shape=(n, 3), contiguous=True)
    check_operand(offsets, "offsets", torch.int64, shape=(n + 1,), contiguous=True)
    check_operand(view, "view", torch.int32, shape=(m,), contiguous=True)
    check_operand(observations, "observations", torch.float64, shape=(m, 2), contiguous=True)
    check_operand(extrinsic, "extrinsic", F32, shape=(V, 3, 4), contiguous=True)
    check_operand(intrinsic, "intrinsic", F32, shape=(V, 3, 3), contiguous=True)
    dev = points.device
    ws = workspace(dev, "ovg_ba_workspace_bytes", V, n, m)
    out = (torch.empty(n, 3, device=dev, dtype=torch.float64), torch.empty(V, 3, 4, device=dev, dtype=torch.float64),
           torch.empty(V, 3, 3, device=dev, dtype=torch.float64), torch.empty(n, device=dev, dtype=torch.float64),
           torch.empty(2, device=dev, dtype=torch.float64), torch.empty(4, device=dev, dtype=torch.int64))
    tr = torch.empty(iterations, device=dev, dtype=torch.float64) if trace else None
    L.check(L.lib().ovg_bundle_adjust(L.ptr(points) if n else None, offsets.data_ptr(), L.ptr(view) if m else None,
                                      L.ptr(observations) if m else None, extrinsic.data_ptr(), intrinsic.data_ptr(), V, n, m,
                                      int(iterations), int(bool(refine_focal)), BA_LOSSES.index(loss), float(loss_scale),
                                      ws.data_ptr(), ws.numel(), *(t.data_ptr() if t.numel() else None for t in out), L.ptr(tr),
                                      L.stream()))
    return out + ((tr,) if trace else ())


def host_read(t: torch.Tensor) -> torch.Tensor:
    """The device-to-host read of a matching or mesh call (its one synchronisation)."""
    return t.cpu()


class Mesher:
    """Triangle mesh (ovg_mesh_*) of F point maps of H x W pixels: ``keep`` uint8 [F*H*W] is the confidence mask (or a caller's
    valid mask); ``images`` fp32 [F,3,H,W] give the colours and the background tests, or None (keep = the mask alone).
    ovg_mesh_count runs here; ``totals`` int64 [3] (reference faces, used vertices, forward faces) is read by the caller, once."""

    def __init__(self, keep: torch.Tensor, images: Optional[torch.Tensor], F: int, H: int, W: int,
                 mask_black_bg: bool = False, mask_white_bg: bool = False):
        check_operand(keep, "keep", torch.uint8, numel=F * H * W, contiguous=True)
        if images is not None:
            check_operand(images, "images", F32, shape=(F, 3, H, W), contiguous=True)
        self.F, self.H, self.W, self.images = F, H, W, images
        dev = keep.device
        self.ws = workspace(dev, "ovg_mesh_workspace_bytes", F, H, W)
        self.totals = torch.zeros(3, device=dev, dtype=torch.int64)
        L.check(L.lib().ovg_mesh_count(keep.data_ptr(), L.ptr(images), F, H, W, int(mask_black_bg), int(mask_white_bg),
                                       self.ws.data_ptr(), self.ws.numel(), self.totals.data_ptr(), L.stream()))

    def faces(self, n: int, colors: Optional[torch.Tensor] = None):
        """The reference layout: (faces int64 [n, 3], face_colors [n, 3]).  Colours: uint8 of ``images``, or gathered from
        ``colors`` [F*H*W, 3] (any dtype of 1, 2, 4 or 8 bytes) into its dtype."""
        dev = self.ws.device
        if colors is None:
            dtype, cptr, cbytes = torch.uint8, None, 1
        else:
            check_operand(colors, "colors", None, numel=self.F * self.H * self.W * 3, contiguous=True)
            dtype, cptr, cbytes = colors.dtype, colors.data_ptr(), colors.element_size()
        faces = torch.empty(max(n, 1), 3, device=dev, dtype=torch.int64)       # >= 1 row: the library wants real pointers
        cols = torch.empty(max(n, 1), 3, device=dev, dtype=dtype)
        L.check(L.lib().ovg_mesh_faces(L.ptr(self.images), cptr, cbytes, self.F, self.H, self.W, self.ws.data_ptr(),
                                       self.ws.numel(), faces.data_ptr(), cols.data_ptr(), L.stream()))
        return faces[:n], cols[:n]

    def compact(self, points: torch.Tensor, n_used: int, n_fwd: int):
        """The GLB layout: (positions fp32 [n_used, 3], colors uint8 [n_used, 3], indices int32 [n_fwd, 3])."""
        if self.images is None:
            raise ValueError("compact needs the images the Mesher was built with")
        check_operand(points, "points", F32, numel=self.F * self.H * self.W * 3, contiguous=True)
        dev = self.ws.device
        pos = torch.empty(max(n_used, 1), 3, device=dev, dtype=F32)
        cols = torch.empty(max(n_used, 1), 3, device=dev, dtype=torch.uint8)
        idx = torch.empty(max(n_fwd, 1), 3, device=dev, dtype=torch.int32)
        L.check(L.lib().ovg_mesh_compact(points.data_ptr(), self.images.data_ptr(), self.F, self.H, self.W, self.ws.data_ptr(),
                                         self.ws.numel(), pos.data_ptr(), cols.data_ptr(), idx.data_ptr(), L.stream()))
        return pos[:n_used], cols[:n_used], idx[:n_fwd]


class Matcher:
    """Reciprocal nearest-neighbour matches (ovg_match_*) between the kept points of V views: points fp32 [V, cap, 3] and keep
    uint8 [V, cap] (or None: all rows), pairs int32 [P, 2] on the device.  Builds every view's index once (ovg_match_index), then
    queries all pairs in both directions (ovg_match_query); ``counts()`` is the one host read."""

    def __init__(self, points: torch.Tensor, keep: Optional[torch.Tensor], pairs: torch.Tensor):
        check_operand(points, "points", F32, shape=(None, None, 3), contiguous=True)
        check_operand(pairs, "pairs", torch.int32, contiguous=True)
        self.V, self.cap = points.shape[0], points.shape[1]
        self.P = pairs.shape[0]
        if keep is not None:
            check_operand(keep, "keep", torch.uint8, numel=self.V * self.cap, contiguous=True)
        self.pairs = pairs
        lib = L.lib()
        self.ws = workspace(points.device, "ovg_match_workspace_bytes", self.V, self.cap, self.P)
        self._counts = torch.zeros(self.P + 1, device=points.device, dtype=torch.int64)
        L.check(lib.ovg_match_index(points.data_ptr(), L.ptr(keep), self.V, self.cap, self.P, self.ws.data_ptr(), self.ws.numel(),
                                    L.stream()))
        L.check(lib.ovg_match_query(pairs.data_ptr(), self.P, self.V, self.cap, self.ws.data_ptr(), self.ws.numel(),
                                    self._counts.data_ptr(), L.stream()))

    def counts(self):
        """(matches per pair as a list of ints, whether a kept point is not finite): the one host read."""
        c = host_read(self._counts).tolist()
        return c[:self.P], bool(c[self.P])

    def gather(self, total: int, W: int):
        """xy_i, xy_j int64 [total, 2]: the matches of all pairs in order (pixel (x, y) = (row % W, row // W))."""
        xy_i = torch.empty(total, 2, device=self.ws.device, dtype=torch.int64)
        xy_j = torch.empty(total, 2, device=self.ws.device, dtype=torch.int64)
        if total:
            L.check(L.lib().ovg_match_gather(self.pairs.data_ptr(), self.P, self.V, self.cap, W, self.ws.data_ptr(), self.ws.numel(),
                                             xy_i.data_ptr(), xy_j.data_ptr(), L.stream()))
        return xy_i, xy_j

    def pair(self, k: int, n_j: int):
        """(reciprocal_in_P2 bool [n_j], nn2_in_P1 int64 [n_j]) of pair k."""
        rec = torch.empty(n_j, device=self.ws.device, dtype=torch.uint8)
        nn = torch.empty(n_j, device=self.ws.device, dtype=torch.int64)
        if n_j:
            L.check(L.lib().ovg_match_pair(self.pairs.data_ptr(), self.P, self.V, self.cap, k, self.ws.data_ptr(), self.ws.numel(),
                                           rec.data_ptr(), nn.data_ptr(), L.stream()))
        return rec.bool(), nn


class Tracker:
    """Star tracks (ovg_tracks_*) over a Matcher's reciprocal matches: the Matcher's pairs must be (i, j) with i < j, unique and
    sorted, and pair_off int32 [V + 1] on the device gives each anchor view's range of them.  Assigns the tracks on
    construction (ovg_tracks_assign); ``counts()`` is the one host read, in place of the Matcher's."""

    def __init__(self, matcher: Matcher, pair_off: torch.Tensor, min_views: int):
        check_operand(pair_off, "pair_off", torch.int32, numel=matcher.V + 1, contiguous=True)
        self.mt = matcher
        dev = matcher.ws.device
        self.ws = workspace(dev, "ovg_tracks_workspace_bytes", matcher.V, matcher.cap)
        self._counts = torch.empty(3, device=dev, dtype=torch.int64)
        L.check(L.lib().ovg_tracks_assign(matcher.pairs.data_ptr(), pair_off.data_ptr(), matcher.P, matcher.V, matcher.cap,
                                          int(min_views), matcher.ws.data_ptr(), matcher.ws.numel(), self.ws.data_ptr(),
                                          self.ws.numel(), self._counts.data_ptr(), L.stream()))

    def counts(self):
        """(tracks, observations, whether a kept point is not finite): the one host read."""
        n, m, bad = host_read(self._counts).tolist()
        return n, m, bool(bad)

    def gather(self, images: torch.Tensor, extrinsic: torch.Tensor, intrinsic: torch.Tensor, W: int, n: int, m: int):
        """The tracks' outputs (ovg_tracks_gather) as a dict of device tensors; images fp32 [V, 3, H, W], extrinsic fp32
        [V, 3, 4], intrinsic fp32 [V, 3, 3], contiguous."""
        mt = self.mt
        check_operand(images, "images", F32, shape=(mt.V, 3, mt.cap // W, W), contiguous=True)
        check_operand(extrinsic, "extrinsic", F32, shape=(mt.V, 3, 4), contiguous=True)
        check_operand(intrinsic, "intrinsic", F32, shape=(mt.V, 3, 3), contiguous=True)
        dev = self.ws.device
        out = {"points": torch.empty(n, 3, device=dev, dtype=torch.float64),
               "colors": torch.empty(n, 3, device=dev, dtype=torch.uint8),
               "error": torch.empty(n, device=dev, dtype=torch.float64),
               "offsets": torch.empty(n + 1, device=dev, dtype=torch.int64),
               "view": torch.empty(m, device=dev, dtype=torch.int32),
               "xy": torch.empty(m, 2, device=dev, dtype=torch.int64),
               "point2d": torch.empty(m, device=dev, dtype=torch.int32),
               "view_offsets": torch.empty(mt.V + 1, device=dev, dtype=torch.int64),
               "view_track": torch.empty(m, device=dev, dtype=torch.int32),
               "view_xy": torch.empty(m, 2, device=dev, dtype=torch.int64)}
        L.check(L.lib().ovg_tracks_gather(
            images.data_ptr(), extrinsic.data_ptr(), intrinsic.data_ptr(), mt.V, mt.cap, mt.P, W, n, m, mt.ws.data_ptr(),
            mt.ws.numel(), self.ws.data_ptr(), self.ws.numel(), *(t.data_ptr() if t.numel() else None for t in out.values()),
            L.stream()))
        return out
