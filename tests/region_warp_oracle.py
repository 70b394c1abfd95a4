"""numpy restatement of the region warp (parseq_warp_regions, regions.cuh) without PIL: Pillow's Geometry.c generic
transform with perspective_transform and bicubic_filter32RGB for an RGB frame, fill 0.  Every float64 operation is a
separate numpy operation in C's evaluation order (numpy never fuses a multiply and an add), so the bytes are PIL's."""
import numpy as np


def _cubic(v1, v2, v3, v4, d):
    """Geometry.c BICUBIC: p1 = v2, p2 = -v1 + v3, p3 = 2 (v1 - v2) + v3 - v4, p4 = -v1 + v2 - v3 + v4, then
    p1 + d (p2 + d (p3 + d p4)).  With integer taps p2..p4 are exact int sums, as in C."""
    if v1.dtype.kind == "i":
        p1 = v2.astype(np.float64)
        p2 = (-v1 + v3).astype(np.float64)
        p3 = (2 * (v1 - v2) + v3 - v4).astype(np.float64)
        p4 = (-v1 + v2 - v3 + v4).astype(np.float64)
    else:
        p1 = v2
        p2 = -v1 + v3
        p3 = 2.0 * (v1 - v2) + v3 - v4
        p4 = -v1 + v2 - v3 + v4
    return p1 + d * (p2 + d * (p3 + d * p4))


def warp(frame: np.ndarray, h: int, w: int, coeffs) -> np.ndarray:
    """frame uint8 [H, W, 3] -> uint8 [h, w, 3]: frame.transform((w, h), PERSPECTIVE, coeffs, BICUBIC)."""
    H, W = frame.shape[:2]
    a0, a1, a2, a3, a4, a5, a6, a7 = (float(c) for c in coeffs)
    yin, xin = np.meshgrid(np.arange(h, dtype=np.float64) + 0.5, np.arange(w, dtype=np.float64) + 0.5, indexing="ij")
    den = a6 * xin + a7 * yin + 1.0
    sx = (a0 * xin + a1 * yin + a2) / den
    sy = (a3 * xin + a4 * yin + a5) / den
    inside = (sx >= 0.0) & (sx < W) & (sy >= 0.0) & (sy < H)
    sx, sy = np.where(inside, sx, 0.5), np.where(inside, sy, 0.5)
    xs, ys = sx - 0.5, sy - 0.5
    ix, iy = np.floor(xs), np.floor(ys)
    dx, dy = xs - ix, ys - iy
    ix, iy = ix.astype(np.int64) - 1, iy.astype(np.int64) - 1
    cols = [np.clip(ix + k, 0, W - 1) for k in range(4)]
    rows = [np.clip(iy + k, 0, H - 1) for k in range(4)]
    out = np.zeros((h, w, 3), dtype=np.uint8)
    for c in range(3):
        v = [_cubic(*(frame[rows[r], cols[k], c].astype(np.int64) for k in range(4)), dx) for r in range(4)]
        o = _cubic(v[0], v[1], v[2], v[3], dy)
        b = np.where(o <= 0.0, 0.0, np.where(o >= 255.0, 255.0, np.trunc(np.clip(o, 0.0, 255.0))))
        out[..., c] = np.where(inside, b, 0.0).astype(np.uint8)
    return out


def pil_warp(frame: np.ndarray, h: int, w: int, coeffs) -> np.ndarray:
    """What PIL itself makes of it (the ground truth the restatement is held to)."""
    from PIL import Image
    img = Image.fromarray(frame, "RGB")
    return np.asarray(img.transform((w, h), Image.Transform.PERSPECTIVE, tuple(float(c) for c in coeffs),
                                    Image.Resampling.BICUBIC))
