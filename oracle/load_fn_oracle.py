"""CPU restatement of the reference's quick-start loader  --  TEST INFRASTRUCTURE (see oracle/omnivggt_oracle.py).

``load_and_preprocess_images`` follows reference omnivggt/utils/load_fn.py:12-146 step by step with numpy: Pillow's bicubic
resize is ``preprocess_oracle.pil_resize_u8`` (the library's published fixed-point arithmetic; tests/test_preprocess.py checks
it against Pillow), ToTensor is uint8 / 255 in float32, and the white padding is ``np.pad`` with 1.0.  Decoding (RGBA on white,
then RGB) is the same Pillow calls the reference makes.  tests/golden/load_fn.json pins it to the unmodified reference.
"""
from __future__ import annotations

from typing import Callable, Sequence

import numpy as np

from oracle.preprocess_oracle import pil_resize_u8

TARGET_SIZE = 518                 # load_fn.py:50


def resized_size(width: int, height: int, mode: str):
    """(new_width, new_height): load_fn.py:70-82."""
    if mode == "pad":
        if width >= height:
            new_width = TARGET_SIZE
            new_height = round(height * (new_width / width) / 14) * 14
        else:
            new_height = TARGET_SIZE
            new_width = round(width * (new_height / height) / 14) * 14
    else:
        new_width = TARGET_SIZE
        new_height = round(height * (new_width / width) / 14) * 14
    return new_width, new_height


def _pad_white(img: np.ndarray, height: int, width: int) -> np.ndarray:
    """[3, h, w] centred in [3, height, width] with 1.0, the extra row / column at the bottom / right: load_fn.py:95-107, :123-134."""
    h_padding, w_padding = height - img.shape[1], width - img.shape[2]
    if h_padding > 0 or w_padding > 0:
        top, left = h_padding // 2, w_padding // 2
        img = np.pad(img, ((0, 0), (top, h_padding - top), (left, w_padding - left)), mode="constant", constant_values=1.0)
    return img


def preprocess_images(images: Sequence[np.ndarray], mode: str = "crop",
                      resize: Callable[[np.ndarray, int, int], np.ndarray] = pil_resize_u8) -> np.ndarray:
    """load_fn.py:39-146 on decoded uint8 RGB images [h, w, 3], in the given order -> float32 [N, 3, H, W].  ``resize`` is
    uint8 [h, w, 3] -> uint8 [new_h, new_w, 3] (Pillow BICUBIC)."""
    if len(images) == 0:
        raise ValueError("At least 1 image is required")
    if mode not in ("crop", "pad"):
        raise ValueError("Mode must be either 'crop' or 'pad'")
    out, shapes = [], set()
    for im in images:
        height, width = im.shape[:2]
        new_width, new_height = resized_size(width, height, mode)
        if new_width <= 0 or new_height <= 0:
            raise ValueError("height and width must be > 0")                       # what Pillow raises at :85
        r = resize(im, new_width, new_height)                                                       # :85
        img = np.ascontiguousarray(r.transpose(2, 0, 1)).astype(np.float32) / np.float32(255)        # :86 ToTensor
        if mode == "crop" and new_height > TARGET_SIZE:                                             # :89-91
            start_y = (new_height - TARGET_SIZE) // 2
            img = img[:, start_y:start_y + TARGET_SIZE, :]
        if mode == "pad":                                                                           # :94-107
            img = _pad_white(img, TARGET_SIZE, TARGET_SIZE)
        shapes.add((img.shape[1], img.shape[2]))
        out.append(img)
    if len(shapes) > 1:                                                                             # :114-136
        max_height = max(s[0] for s in shapes)
        max_width = max(s[1] for s in shapes)
        out = [_pad_white(img, max_height, max_width) for img in out]
    return np.stack(out)


def decode(path: str) -> np.ndarray:
    """load_fn.py:56-66: open, composite RGBA on white, convert to RGB."""
    from PIL import Image
    img = Image.open(path)
    if img.mode == "RGBA":
        img = Image.alpha_composite(Image.new("RGBA", img.size, (255, 255, 255, 255)), img)
    return np.asarray(img.convert("RGB"))


def load_and_preprocess_images(image_path_list: Sequence[str], mode: str = "crop") -> np.ndarray:
    """load_fn.py:12-146: the paths are sorted (:51), decoded, then preprocessed."""
    if len(image_path_list) == 0:
        raise ValueError("At least 1 image is required")
    return preprocess_images([decode(p) for p in sorted(image_path_list)], mode)
