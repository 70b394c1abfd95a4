"""CPU oracle of the engine's raw-crop preprocessing (parseq_b200/csrc/crops.cuh): the reference's
`SceneTextDataModule.get_transform(img_size, rotation=r)` (strhub/data/module.py:69-82) restated in numpy, without PIL.

- rotation r in {0, 90, 180, 270}: `Image.rotate(r, expand=True)` == `np.rot90(crop, r // 90)` (counter-clockwise);
- `T.Resize(img_size, BICUBIC)` == PIL's uint8 `Image.resize`: two separable passes with uint8 between them, each output
  value clip8((2^21 + sum in * k) >> 22) with the 22-bit fixed-point coefficients of Resample.c (precompute_coeffs,
  normalize_coeffs_8bpc); horizontal first, except that `Image.resize` runs the vertical pass first when
  h > 100 w and the height shrinks; a pass whose axis keeps its size is skipped;
- `ToTensor` + `Normalize(0.5, 0.5)`: (u8 / 255 - 0.5) / 0.5 in float32.
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np

PRECISION_BITS = 22
MAX_SIDE = 8192


def _cubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0
    if x < 2.0:
        return (((x - 5.0) * x + 8.0) * x - 4.0) * a
    return 0.0


def coeffs(in_size: int, out_size: int) -> List[Tuple[int, List[int]]]:
    """(xmin, fixed-point taps) of every output coordinate of an in_size -> out_size pass (Python floats are IEEE
    doubles, evaluated without fused multiply-add, as PIL's C is)."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ss = 1.0 / fs
    out = []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_cubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:                      # in tap order
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        k = [int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS)) for v in w]
        out.append((xmin, k))
    return out


def resample_axis(img: np.ndarray, out_size: int, axis: int) -> np.ndarray:
    """One uint8 bicubic pass along `axis` (0 = vertical, 1 = horizontal) of an HWC uint8 image."""
    in_size = img.shape[axis]
    if in_size == out_size:
        return img
    a = np.moveaxis(img, axis, 0).astype(np.int64)
    res = np.empty((out_size,) + a.shape[1:], np.int64)
    for i, (xmin, k) in enumerate(coeffs(in_size, out_size)):
        kk = np.asarray(k, np.int64).reshape((-1,) + (1,) * (a.ndim - 1))
        acc = (1 << (PRECISION_BITS - 1)) + (a[xmin:xmin + len(k)] * kk).sum(axis=0)
        acc = ((acc + 2 ** 31) % 2 ** 32) - 2 ** 31        # int32 accumulator, as PIL's
        res[i] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(res.astype(np.uint8), 0, axis)


def resize_bicubic(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """PIL `Image.fromarray(img).resize((out_w, out_h), BICUBIC)` of a uint8 [h, w, 3] array."""
    h, w = img.shape[:2]
    if h > w * 100 and out_h < h:
        return resample_axis(resample_axis(img, out_h, 0), out_w, 1)
    return resample_axis(resample_axis(img, out_w, 1), out_h, 0)


def rotate(img: np.ndarray, rotation: int) -> np.ndarray:
    if rotation not in (0, 90, 180, 270):
        raise ValueError("rotation must be 0, 90, 180 or 270")
    return np.ascontiguousarray(np.rot90(img, rotation // 90))


def transform_u8(img: np.ndarray, img_size: Tuple[int, int], rotation: int = 0) -> np.ndarray:
    """uint8 [H, W, 3]: rotate, then resize to img_size = (H, W)."""
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise ValueError("crop must be uint8 [h, w, 3]")
    return resize_bicubic(rotate(img, rotation), int(img_size[0]), int(img_size[1]))


def to_float(u8: np.ndarray) -> np.ndarray:
    """ToTensor + Normalize(0.5, 0.5): float32 [3, H, W]."""
    x = u8.astype(np.float32).transpose(2, 0, 1) / np.float32(255)
    return (x - np.float32(0.5)) / np.float32(0.5)


def transform(img: np.ndarray, img_size: Tuple[int, int], rotation: int = 0) -> np.ndarray:
    """The reference's whole test-time transform of one crop: float32 [3, H, W]."""
    return to_float(transform_u8(img, img_size, rotation))

