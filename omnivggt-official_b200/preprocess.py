"""GPU input pipeline: drop-in for reference ``visual_util.load_images_and_cameras`` (visual_util.py:679-841).

Baseline JPEGs (what cameras and phones write) are decoded on the device, bit-identical to Pillow (``decode_images``,
csrc/jpeg.cuh); every other file (PNG, progressive JPEG, CMYK, ...) and .npy / camera .txt parsing stays on the host, and
RGBA is composited on white there.  Everything the reference
then does per view with Pillow / OpenCV / numpy -- bicubic resize to width 518, height to a multiple of 14, centre crop, ToTensor,
depth validity filter + nearest resize + crop + mask, intrinsics rescale, camera-to-world -> world-to-camera -- runs in libovg
kernels on the device and returns the model's input tuple as CUDA tensors.  The small per-size tap / index tables are computed on
the host with the arithmetic the two libraries publish (Pillow Resample.c, OpenCV resizeNN) and cached on the device, so the image
tensor equals the reference's bit for bit (tests/test_preprocess.py compares against Pillow / OpenCV and the reference loader).

``load_and_preprocess_images`` / ``preprocess_images`` are the same for the reference's quick-start loader
(omnivggt/utils/load_fn.py:12-146): crop or pad mode, and lists of mixed image sizes padded with white to the largest shape,
written straight into the output frame by the resize kernel (tests/test_load_fn.py)."""
from __future__ import annotations

import ctypes
import glob
import math
import os
from pathlib import Path
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L

PRECISION_BITS = 32 - 8 - 2
_tables: Dict[tuple, tuple] = {}


def target_geometry(width: int, height: int, target_size: int = 518) -> Tuple[int, int, int, int]:
    """(new_width, new_height, crop_start_y, final_height)   -- visual_util.py:731-747."""
    new_width = target_size
    new_height = round(height * (new_width / width) / 14) * 14
    crop = (new_height - target_size) // 2 if new_height > target_size else 0
    return new_width, new_height, crop, min(new_height, target_size)


def _bicubic(x: float) -> float:
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def bicubic_taps(in_size: int, out_size: int, device) -> tuple:
    """Pillow's fixed-point bicubic taps of one axis as device tensors (kmin, kcnt, kk [out, ksize], ksize)."""
    key = ("bicubic", in_size, out_size, str(device))
    if key not in _tables:
        scale = in_size / out_size
        filterscale = max(scale, 1.0)
        support = 2.0 * filterscale
        ksize = int(math.ceil(support)) * 2 + 1
        kmin, kcnt = np.zeros(out_size, np.int32), np.zeros(out_size, np.int32)
        kk = np.zeros((out_size, ksize), np.int32)
        ss = 1.0 / filterscale
        for xx in range(out_size):
            center = (xx + 0.5) * scale
            lo = max(int(center - support + 0.5), 0)
            hi = min(int(center + support + 0.5), in_size)
            w = [_bicubic((x + lo - center + 0.5) * ss) for x in range(hi - lo)]
            ww = sum(w)
            if ww != 0.0:
                w = [v / ww for v in w]
            for x, v in enumerate(w):
                kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
            kmin[xx], kcnt[xx] = lo, hi - lo
        _tables[key] = (torch.from_numpy(kmin).to(device), torch.from_numpy(kcnt).to(device), torch.from_numpy(kk).to(device), ksize)
    return _tables[key]


def nearest_index(src: int, dst: int, device) -> torch.Tensor:
    """Source index per destination index of cv2.resize(..., INTER_NEAREST)."""
    key = ("nearest", src, dst, str(device))
    if key not in _tables:
        inv = 1.0 / (dst / src)
        idx = np.minimum(np.floor(np.arange(dst) * inv).astype(np.int64), src - 1).astype(np.int32)
        _tables[key] = (torch.from_numpy(idx).to(device),)
    return _tables[key][0]


def decode_rgb(path: str) -> np.ndarray:
    """uint8 RGB [h, w, 3] of an image file; RGBA is composited on white first (visual_util.py:722-726, load_fn.py:59-66)."""
    from PIL import Image
    img = Image.open(path)
    if img.mode == "RGBA":
        img = Image.alpha_composite(Image.new("RGBA", img.size, (255, 255, 255, 255)), img)
    return np.asarray(img.convert("RGB"))


@torch.no_grad()
def decode_images(paths: Sequence[str], device="cuda", subseq_bits: int = 0) -> List[torch.Tensor]:
    """uint8 RGB [h, w, 3] tensors on `device`, in the given order, equal to ``decode_rgb`` bit for bit.  One plan for the list,
    one pinned host-to-device copy of its staging stream and one ``ovg_jpeg_decode`` for every baseline JPEG; ``decode_rgb``
    (Pillow) and an upload for the other files and for any file the device flags (inconsistent entropy data, or a block
    outside the range where libjpeg-turbo's C and SIMD IDCTs agree).  subseq_bits: bits per
    subsequence of the parallel Huffman decoder (0: the default, 512)."""
    paths = list(paths)
    dev = torch.device(device)
    data = [Path(p).read_bytes() for p in paths]
    plan = L.JpegPlan(data, subseq_bits)
    out: List[Optional[torch.Tensor]] = [None] * len(paths)
    on_device = [i for i, f in enumerate(plan.files) if f[0] == L.JPEG_DEVICE]
    if on_device:
        lib = L.lib()
        staging = torch.empty(plan.stream_bytes, dtype=torch.uint8, pin_memory=dev.type == "cuda")
        plan.fill_stream(staging.data_ptr())
        stream = staging.to(dev, non_blocking=True)
        ws = torch.empty(plan.workspace_bytes, dtype=torch.uint8, device=dev)
        st = torch.zeros(len(paths), dtype=torch.int32, device=dev)
        ptrs = (ctypes.c_void_p * len(paths))()
        for i in on_device:
            _, h, w, _ = plan.files[i]
            out[i] = torch.empty(h, w, 3, dtype=torch.uint8, device=dev)
            ptrs[i] = out[i].data_ptr()
        L.check(lib.ovg_jpeg_decode(plan.handle, stream.data_ptr(), ptrs, st.data_ptr(), ws.data_ptr(), plan.workspace_bytes,
                                    L.stream()))
    for i, p in enumerate(paths):                  # overlaps the scan, IDCT and colour kernels (not the sync rounds)
        if out[i] is None:
            out[i] = torch.from_numpy(np.array(decode_rgb(p))).to(dev)
    if on_device:
        status = st.cpu()                          # synchronises: the staging buffers are free after this
        for i in on_device:
            if int(status[i]):
                out[i] = torch.from_numpy(np.array(decode_rgb(paths[i]))).to(dev)
    return out


def _resize_view(lib, st, im, nw: int, nh: int, crop: int, fh: int, out: torch.Tensor, dev, frame=None, fill: float = 1.0) -> list:
    """Upload one uint8 RGB view [h, w, 3] and launch its bicubic resize to [nh, nw], rows [crop, crop + fh) and ToTensor into
    out [3, fh, nw]; with frame = (out_h, out_w, off_y, off_x), into the frame out [3, out_h, out_w] at that offset, the rest
    set to fill.  Returns the staging tensors, which must stay alive until the launches have run."""
    h, w = int(im.shape[0]), int(im.shape[1])
    src = torch.as_tensor(np.array(im, dtype=np.uint8, copy=True) if isinstance(im, np.ndarray) else im, dtype=torch.uint8).to(dev).contiguous()
    if src.shape != (h, w, 3):
        raise ValueError(f"images are uint8 RGB [h, w, 3], got {list(src.shape)}")
    hk = bicubic_taps(w, nw, dev) if w != nw else (None, None, None, 0)
    vk = bicubic_taps(h, nh, dev) if h != nh else (None, None, None, 0)
    tmp = torch.empty(h, nw, 3, device=dev, dtype=torch.uint8) if w != nw else None
    args = (src.data_ptr(), h, w, nw, nh, crop, fh, L.ptr(hk[0]), L.ptr(hk[1]), L.ptr(hk[2]), hk[3], L.ptr(vk[0]), L.ptr(vk[1]),
            L.ptr(vk[2]), vk[3], L.ptr(tmp), out.data_ptr())
    if frame is None:
        L.check(lib.ovg_preprocess_image(*args, st))
    else:
        L.check(lib.ovg_preprocess_image_canvas(*args, *frame, float(fill), st))
    return [src, tmp]


@torch.no_grad()
def preprocess_views(images: Sequence, cameras: Optional[Sequence] = None, depths: Optional[Sequence] = None,
                     target_size: int = 518, max_depth: float = 100.0, device="cuda", depth_transposed: Optional[Sequence[bool]] = None):
    """images: uint8 RGB arrays / tensors [h, w, 3]; cameras: per view (camera-to-world 3x4 or 4x4, K 3x3) or None; depths: per view
    float32 [h', w'] as loaded or None.  Returns (images [S,3,H,W], extrinsics [1,S,3,4], intrinsics [1,S,3,3], depth [1,S,H,W,1],
    mask [1,S,H,W], depth_indices, camera_indices) -- CUDA tensors, the tuple reference visual_util.py:835-841 returns."""
    lib = L.lib()
    dev = torch.device(device)
    S = len(images)
    cameras = list(cameras) if cameras is not None else [None] * S
    depths = list(depths) if depths is not None else [None] * S
    depth_transposed = list(depth_transposed) if depth_transposed is not None else [False] * S
    geoms = []
    for im in images:
        h, w = int(im.shape[0]), int(im.shape[1])
        geoms.append((h, w) + target_geometry(w, h, target_size))
    fh, nw = geoms[0][5], geoms[0][2]
    if any(g[5] != fh for g in geoms):
        raise ValueError("all views of a scene must resize to the same height (the reference stacks them: visual_util.py:835)")
    out = torch.empty(S, 3, fh, nw, device=dev, dtype=torch.float32)
    dmap = torch.zeros(S, fh, nw, device=dev, dtype=torch.float32)
    mask = torch.zeros(S, fh, nw, device=dev, dtype=torch.float32)
    c2w = torch.zeros(S, 3, 4, dtype=torch.float32)
    kin = torch.zeros(S, 3, 3, dtype=torch.float32)
    geom = torch.zeros(S, 3, dtype=torch.float32)
    has = torch.zeros(S, dtype=torch.int32)
    didx, cidx = [], []
    st = L.stream()
    keep = []
    for i, (im, (h, w, _, nh, crop, _)) in enumerate(zip(images, geoms)):
        keep += _resize_view(lib, st, im, nw, nh, crop, fh, out[i], dev)
        dep = depths[i]
        if dep is not None:
            d = torch.as_tensor(np.ascontiguousarray(dep, dtype=np.float32) if isinstance(dep, np.ndarray) else dep).float().to(dev).contiguous()
            rows, cols = d.shape
            if depth_transposed[i]:         # the reference transposes PNG depth maps after reading them (visual_util.py:771)
                sh, sw, rs, cs = cols, rows, 1, cols
            else:
                sh, sw, rs, cs = rows, cols, cols, 1
            L.check(lib.ovg_preprocess_depth(d.data_ptr(), rs, cs, nearest_index(sh, nh, dev).data_ptr(),
                                             nearest_index(sw, nw, dev).data_ptr(), crop, fh, nw, float(max_depth),
                                             dmap[i].data_ptr(), mask[i].data_ptr(), st))
            keep.append(d)
            didx.append(i)
        cam = cameras[i]
        if cam is not None:
            e, k = np.asarray(cam[0], np.float32), np.asarray(cam[1], np.float32)
            c2w[i] = torch.from_numpy(e[:3, :4].copy())
            kin[i] = torch.from_numpy(k.copy())
            geom[i] = torch.tensor([np.float32(nw / w), np.float32(nh / h), float(crop) if nh > target_size else -1.0])
            has[i] = 1
            cidx.append(i)
    w2c = torch.empty(S, 3, 4, device=dev, dtype=torch.float32)
    kout = torch.empty(S, 3, 3, device=dev, dtype=torch.float32)
    c2w_d, kin_d, geom_d, has_d = c2w.to(dev), kin.to(dev), geom.to(dev), has.to(dev)
    L.check(lib.ovg_prepare_cameras(c2w_d.data_ptr(), kin_d.data_ptr(), geom_d.data_ptr(), has_d.data_ptr(), w2c.data_ptr(),
                                    kout.data_ptr(), S, st))
    torch.cuda.current_stream().synchronize()     # the staging tensors in `keep` are released after the kernels ran
    return out, w2c[None], kout[None], dmap[None, ..., None], mask[None], didx, cidx


def read_camera_txt(path: str):
    """3 lines 3x4 camera-to-world + 3 lines 3x3 K, '#' comments allowed (visual_util.py:843-891)."""
    try:
        lines = [ln.strip() for ln in open(path) if ln.strip() and not ln.strip().startswith("#")]
        if len(lines) < 6:
            return None
        e = [[float(x) for x in lines[i].split()] for i in range(3)]
        k = [[float(x) for x in lines[i].split()] for i in range(3, 6)]
        if any(len(r) != 4 for r in e) or any(len(r) != 3 for r in k):
            return None
        return np.array(e, np.float32), np.array(k, np.float32)
    except Exception:
        return None


def load_images_and_cameras(image_folder: str, camera_folder: Optional[str] = None, depth_folder: Optional[str] = None,
                            target_size: int = 518, max_depth: float = 100, device="cuda"):
    """Same signature, file layout and return tuple as reference visual_util.load_images_and_cameras (visual_util.py:679-841);
    images are decoded by ``decode_images`` (baseline JPEGs on the device), depth maps and cameras on the host, the rest runs
    on the GPU."""
    from PIL import Image
    paths = sorted(glob.glob(os.path.join(image_folder, "*")))
    paths = [p for p in paths if p.lower().endswith((".png", ".jpg", ".jpeg"))]
    images = decode_images(paths, device)
    cams, deps, transposed = [], [], []
    for p in paths:
        stem = Path(p).stem
        dep, tr = None, False
        if depth_folder is not None:
            for cand in (os.path.join(depth_folder, stem + ".npy"), os.path.join(depth_folder, stem + ".png")):
                if os.path.exists(cand):                         # both present: the later candidate wins, as in the reference loop
                    if cand.endswith(".npy"):
                        dep, tr = np.load(cand).astype(np.float32), False
                    else:
                        dep, tr = np.asarray(Image.open(cand)).astype(np.float32), True
        deps.append(dep)
        transposed.append(tr)
        cam = None
        if camera_folder is not None and os.path.exists(os.path.join(camera_folder, stem + ".txt")):
            cam = read_camera_txt(os.path.join(camera_folder, stem + ".txt"))
        cams.append(cam)
    return preprocess_views(images, cams, deps, target_size, max_depth, device, transposed)


LOAD_FN_SIZE = 518           # load_fn.py:50; fixed in the reference


def _check_load_fn_args(n: int, mode: str) -> None:
    if n == 0:
        raise ValueError("At least 1 image is required")
    if mode not in ("crop", "pad"):
        raise ValueError("Mode must be either 'crop' or 'pad'")


def load_fn_layout(sizes: Sequence[Tuple[int, int]], mode: str = "crop"):
    """Geometry of reference load_and_preprocess_images (load_fn.py:68-136) for images of sizes [(h, w)].
    Returns (views, (H, W), shapes): per image (new_width, new_height, crop_start_y, kept_height, off_y, off_x), where
    off_* is where its [kept_height, new_width] pixels sit in the output frame [H, W]; and the set of shapes before the
    mixed-size padding, in the reference's insertion order (it prints that set).  Raises ValueError before any device work."""
    _check_load_fn_args(len(sizes), mode)
    T = LOAD_FN_SIZE
    first, shapes = [], set()
    for h, w in sizes:
        if mode == "pad" and h > w:                 # :75-77 the height is the longer side: it becomes 518
            nw, nh = round(w * (T / h) / 14) * 14, T
            crop, fh = 0, nh
        else:                                       # :72-74, :78-82 the width becomes 518; crop mode keeps 518 rows (:89-91)
            nw, nh, crop, fh = target_geometry(w, h, T)
        if nw <= 0 or nh <= 0:
            raise ValueError(f"a {w}x{h} image resizes to {nw}x{nh}: height and width must be > 0")
        if mode == "pad":                           # :94-107 centred in 518 x 518
            top, left, shape = (T - fh) // 2, (T - nw) // 2, (T, T)
        else:
            top, left, shape = 0, 0, (fh, nw)
        first.append((nw, nh, crop, fh, top, left, shape))
        shapes.add(shape)
    H, W = max(s[0] for s in shapes), max(s[1] for s in shapes)
    # :114-136 a second centring pad to the largest shape; the offset is the sum of both pads, each rounded down on its own
    views = [(nw, nh, crop, fh, top + (H - s[0]) // 2, left + (W - s[1]) // 2) for nw, nh, crop, fh, top, left, s in first]
    return views, (H, W), shapes


@torch.no_grad()
def preprocess_images(images: Sequence, mode: str = "crop", device="cuda") -> torch.Tensor:
    """Reference load_and_preprocess_images (load_fn.py:12-146) on decoded images: uint8 RGB arrays / tensors [h, w, 3], in
    the given order.  Returns CUDA fp32 [N, 3, H, W], bit-identical to the reference: Pillow-exact bicubic resize, crop or
    white (1.0) padding to 518 x 518, then white padding of mixed sizes to the largest shape, each view in one libovg call."""
    views, (H, W), shapes = load_fn_layout([(int(im.shape[0]), int(im.shape[1])) for im in images], mode)
    if len(shapes) > 1:
        print(f"Warning: Found images with different shapes: {shapes}")
    lib = L.lib()
    dev = torch.device(device)
    out = torch.empty(len(views), 3, H, W, device=dev, dtype=torch.float32)
    st = L.stream()
    keep = []
    for i, (im, (nw, nh, crop, fh, off_y, off_x)) in enumerate(zip(images, views)):
        keep += _resize_view(lib, st, im, nw, nh, crop, fh, out[i], dev, frame=(H, W, off_y, off_x), fill=1.0)
    torch.cuda.current_stream().synchronize()     # the staging tensors in `keep` are released after the kernels ran
    return out


def load_and_preprocess_images(image_path_list: Sequence[str], mode: str = "crop", device="cuda") -> torch.Tensor:
    """Same signature (plus device) and result as reference omnivggt.utils.load_fn.load_and_preprocess_images: the paths are
    sorted and decoded by ``decode_images`` (baseline JPEGs on the device, other files with Pillow, RGBA on white), the rest
    runs on the GPU (preprocess_images)."""
    _check_load_fn_args(len(image_path_list), mode)
    return preprocess_images(decode_images(sorted(image_path_list), device), mode, device)
