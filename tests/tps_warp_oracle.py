"""fp64 restatement of the curved-region warp (parseq_warp_polygons, region_tps_kernel) in numpy: the thin-plate spline
of include/parseq_b200.h in its order, with numpy's log, fed the coefficients of parseq_tps_coeffs, then the sampler tail
of region_warp_oracle.py (its Geometry.c BICUBIC `_cubic`, at given frame points; test_curved_regions_cpu.py holds it
to region_warp_oracle.warp on the quad goldens).  numpy never fuses a multiply and an add, so every operation but ln is the kernel's to the bit.
The device's ln may differ from numpy's in the last bits, so a byte is only held to the restatement where it does not
change when the mapped point moves by 1e-7 px (`fragile`)."""
import numpy as np

from region_warp_oracle import _cubic

EPS = 1e-7                                  # px: a move that dwarfs any ln rounding difference in the map


def sample(frame: np.ndarray, sx: np.ndarray, sy: np.ndarray) -> np.ndarray:
    """region_warp_oracle.warp's tail at frame points (sx, sy) float64 [h, w] -> uint8 [h, w, 3]: 0 outside
    [0, W) x [0, H), else 0.5 subtracted, the floor taken, Geometry.c's BICUBIC rows first with clamped taps, clipped
    and truncated."""
    H, W = frame.shape[:2]
    h, w = sx.shape
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


def tps_map(tps, h: int, w: int):
    """(X, Y) float64 [h, w]: frame points of the output pixels of an h x w crop under TPS coefficients [F + 3][2]."""
    t = np.asarray(tps, dtype=np.float64)
    k = (t.shape[0] - 3) // 2
    cx = np.linspace(-1.0, 1.0, k)
    xn = (np.arange(-w, w, 2) + 1.0) / w     # _build_P
    yn = (np.arange(-h, h, 2) + 1.0) / h
    yn, xn = np.meshgrid(yn, xn, indexing="ij")
    X = t[0, 0] + t[1, 0] * xn + t[2, 0] * yn
    Y = t[0, 1] + t[1, 1] * xn + t[2, 1] * yn
    for m in range(2 * k):
        dx, dy = xn - cx[m % k], yn - (-1.0 if m < k else 1.0)
        r = np.sqrt(dx * dx + dy * dy)
        phi = (r * r) * np.log(r + 1e-6)
        X = X + t[3 + m, 0] * phi
        Y = Y + t[3 + m, 1] * phi
    return X, Y


def warp(frame: np.ndarray, h: int, w: int, tps) -> np.ndarray:
    """frame uint8 [H, W, 3] -> uint8 [h, w, 3], the crop of the polygon with TPS coefficients tps."""
    X, Y = tps_map(tps, h, w)
    return sample(frame, X, Y)


def fragile(frame: np.ndarray, h: int, w: int, tps) -> np.ndarray:
    """bool [h, w]: pixels whose bytes change when the mapped point moves by EPS along x or y."""
    X, Y = tps_map(tps, h, w)
    base = sample(frame, X, Y)
    out = np.zeros((h, w), dtype=bool)
    for ddx, ddy in ((EPS, 0.0), (-EPS, 0.0), (0.0, EPS), (0.0, -EPS)):
        out |= (sample(frame, X + ddx, Y + ddy) != base).any(-1)
    return out
