"""Geometry of text regions (parseq_warp_regions): a quadrilateral of frame pixels -> the size of its rectified crop and
the 8 coefficients of PIL's PERSPECTIVE transform that map the crop onto it.  Pure Python doubles, so the coefficients
are the same bits on every host.

A region is 4 corners in reading order, TL, TR, BR, BL (ICDAR 2015 / DBNet order), in frame pixels where pixel i covers
[i, i + 1).  Its crop is w = max(1, floor(max(|TR - TL|, |BR - BL|) + 0.5)) wide and h = max(1, floor(max(|BL - TL|,
|BR - TR|) + 0.5)) tall.  The map is Heckbert's closed-form square-to-quad projective map (its affine branch when
x0 - x1 + x2 - x3 == 0 and y0 - y1 + y2 - y3 == 0) composed with s = u / w, t = v / h, so that crop points (0, 0),
(w, 0), (w, h) and (0, h) go to TL, TR, BR and BL: x = (a0 u + a1 v + a2) / (a6 u + a7 v + 1), likewise y."""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

MAX_SIDE = 8192        # crop sides: the raw-crop path's limit

Quad = Sequence[Sequence[float]]


def quad_size(q: Quad) -> Tuple[int, int]:
    """(h, w) of the crop of quad q = (TL, TR, BR, BL)."""
    (x0, y0), (x1, y1), (x2, y2), (x3, y3) = [(float(p[0]), float(p[1])) for p in q]
    w = max(math.hypot(x1 - x0, y1 - y0), math.hypot(x2 - x3, y2 - y3))
    h = max(math.hypot(x3 - x0, y3 - y0), math.hypot(x2 - x1, y2 - y1))
    return max(1, math.floor(h + 0.5)), max(1, math.floor(w + 0.5))


def quad_coeffs(q: Quad, h: int, w: int) -> Tuple[float, ...]:
    """PIL PERSPECTIVE coefficients (a0..a7) that send crop (0, 0), (w, 0), (w, h), (0, h) to TL, TR, BR, BL."""
    (x0, y0), (x1, y1), (x2, y2), (x3, y3) = [(float(p[0]), float(p[1])) for p in q]
    px = x0 - x1 + x2 - x3
    py = y0 - y1 + y2 - y3
    if px == 0.0 and py == 0.0:                     # parallelogram: affine
        a, b, c = x1 - x0, x2 - x1, x0
        d, e, f = y1 - y0, y2 - y1, y0
        g = hh = 0.0
    else:
        dx1, dx2 = x1 - x2, x3 - x2
        dy1, dy2 = y1 - y2, y3 - y2
        det = dx1 * dy2 - dx2 * dy1
        g = (px * dy2 - dx2 * py) / det
        hh = (dx1 * py - px * dy1) / det
        a, b, c = x1 - x0 + g * x1, x3 - x0 + hh * x3, x0
        d, e, f = y1 - y0 + g * y1, y3 - y0 + hh * y3, y0
    w, h = float(w), float(h)
    return (a / w, b / h, c, d / w, e / h, f, g / w, hh / h)


def box_quad(box: Sequence[int]) -> List[Tuple[float, float]]:
    """An integer box (x0, y0, x1, y1) as the quad TL, TR, BR, BL."""
    x0, y0, x1, y1 = (int(v) for v in box)
    return [(float(x0), float(y0)), (float(x1), float(y0)), (float(x1), float(y1)), (float(x0), float(y1))]


def check_quad(q: Quad, i: int = 0):
    """ValueError unless q is 4 finite corners of a strictly convex quadrilateral (either winding), crop sides <= 8192."""
    pts = [(float(p[0]), float(p[1])) for p in q]
    if not all(math.isfinite(v) for p in pts for v in p):
        raise ValueError(f"region {i}: non-finite corner")
    turns = []
    for k in range(4):
        (ax, ay), (bx, by), (cx, cy) = pts[k], pts[(k + 1) % 4], pts[(k + 2) % 4]
        turns.append((bx - ax) * (cy - by) - (by - ay) * (cx - bx))
    if not (all(t > 0.0 for t in turns) or all(t < 0.0 for t in turns)):
        raise ValueError(f"region {i}: the quad {pts} is degenerate, self-intersecting or not convex")
    h, w = quad_size(pts)
    if h > MAX_SIDE or w > MAX_SIDE:
        raise ValueError(f"region {i}: crop size {h} x {w}, sides must be at most {MAX_SIDE}")


def map_points(coeffs: Sequence[float], u, v):
    """Crop points (u, v) -> frame points (x, y) through the coefficients (numbers, arrays or tensors)."""
    a0, a1, a2, a3, a4, a5, a6, a7 = coeffs
    den = a6 * u + a7 * v + 1.0
    return (a0 * u + a1 * v + a2) / den, (a3 * u + a4 * v + a5) / den


# ---------------------------------------------------------------- curved regions (parseq_warp_polygons)
# A polygon of 2k points, 3 <= k <= 32, in the Total-Text / CTW1500 clockwise order: the top edge p_0..p_{k-1} left to
# right, then the bottom edge q_0..q_{k-1} right to left.  The engine takes TRBA's fiducial order, both edges left to
# right: C'_j = p_j, C'_{k+j} = b_j = q_{k-1-j}.  The crop is w = max(1, floor(max(sum |p_{j+1} - p_j|,
# sum |b_{j+1} - b_j|) + 0.5)) wide and h = max(1, floor(max_j |p_j - b_j| + 0.5)) tall; with k = 2 that is quad_size.
# The map is the thin-plate spline of include/parseq_b200.h (parseq_tps_coeffs, map_tps).
MIN_K, MAX_K = 3, 32


def engine_points(poly: Quad) -> List[Tuple[float, float]]:
    """Caller order (top left to right, bottom right to left) -> engine order (both edges left to right)."""
    pts = [(float(p[0]), float(p[1])) for p in poly]
    k = len(pts) // 2
    return pts[:k] + pts[k:][::-1]


def polygon_size(points: Quad) -> Tuple[int, int]:
    """(h, w) of the crop of a polygon given in engine order (top then bottom, each left to right)."""
    pts = [(float(p[0]), float(p[1])) for p in points]
    k = len(pts) // 2
    top, bot = pts[:k], pts[k:]
    lt = lb = hh = 0.0
    for j in range(k - 1):
        lt += math.hypot(top[j + 1][0] - top[j][0], top[j + 1][1] - top[j][1])
        lb += math.hypot(bot[j + 1][0] - bot[j][0], bot[j + 1][1] - bot[j][1])
    for j in range(k):
        hh = max(hh, math.hypot(bot[j][0] - top[j][0], bot[j][1] - top[j][1]))
    return max(1, math.floor(hh + 0.5)), max(1, math.floor(max(lt, lb) + 0.5))


def check_polygon(poly: Quad, i: int = 0):
    """ValueError unless poly (caller order) is 6..64 finite points, an even count, of a simple polygon (no zero-length
    edge, no two edges that meet other than adjacent ones at their shared point), crop sides <= 8192."""
    import numpy as np
    n = len(poly)
    if n % 2 or n < 2 * MIN_K or n > 2 * MAX_K:
        raise ValueError(f"region {i}: {n} points, a polygon needs an even count of 6 to 64 points")
    p = np.asarray([(float(a[0]), float(a[1])) for a in poly], dtype=np.float64)
    if not np.isfinite(p).all():
        raise ValueError(f"region {i}: non-finite point")
    a, b = p, np.roll(p, -1, axis=0)                     # edge e = (a[e], b[e]), the closed boundary
    d = b - a
    if ((d[:, 0] == 0.0) & (d[:, 1] == 0.0)).any():
        raise ValueError(f"region {i}: the polygon is degenerate (a repeated point)")

    def orient(o, u, v):                                  # cross(u - o, v - o) over all (edge, edge) pairs
        return (u[..., 0] - o[..., 0]) * (v[..., 1] - o[..., 1]) - (u[..., 1] - o[..., 1]) * (v[..., 0] - o[..., 0])
    A, B, Cq, D = a[:, None], b[:, None], a[None, :], b[None, :]
    o1, o2, o3, o4 = orient(A, B, Cq), orient(A, B, D), orient(Cq, D, A), orient(Cq, D, B)
    col = (o1 == 0.0) & (o2 == 0.0)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    # overlapping bounding boxes: needed for any meeting, and what decides it for (nearly) collinear edges
    overlap = ((np.maximum(lo[:, None], lo[None, :]) <= np.minimum(hi[:, None], hi[None, :])).all(-1))
    meet = (o1 * o2 <= 0.0) & (o3 * o4 <= 0.0) & overlap
    e = np.arange(n)
    gap = (e[None, :] - e[:, None]) % n
    nonadjacent = (gap >= 2) & (gap <= n - 2)
    # adjacent edges may only share their point: folding back along the same line is a self-intersection
    fold = (gap == 1) & col & ((d[:, None] * d[None, :]).sum(-1) < 0.0)
    if (meet & nonadjacent).any() or fold.any():
        raise ValueError(f"region {i}: the polygon is self-intersecting")
    h, w = polygon_size(engine_points(poly))
    if h > MAX_SIDE or w > MAX_SIDE:
        raise ValueError(f"region {i}: crop size {h} x {w}, sides must be at most {MAX_SIDE}")


def map_tps(tps, h: int, w: int, u, v):
    """Crop points (u, v) of an h x w crop -> frame points (x, y) through the TPS coefficients tps [F + 3][2]: xn =
    2u / w - 1, yn = 2v / h - 1, then the map of include/parseq_b200.h in its order (float64 tensors)."""
    import numpy as np
    import torch
    t = torch.as_tensor(tps, dtype=torch.float64)
    k = (t.shape[0] - 3) // 2
    cx = torch.from_numpy(np.linspace(-1.0, 1.0, k))
    xn = 2.0 * torch.as_tensor(u, dtype=torch.float64) / w - 1.0
    yn = 2.0 * torch.as_tensor(v, dtype=torch.float64) / h - 1.0
    x = t[0, 0] + t[1, 0] * xn + t[2, 0] * yn
    y = t[0, 1] + t[1, 1] * xn + t[2, 1] * yn
    for m in range(2 * k):
        dx, dy = xn - cx[m % k], yn - (-1.0 if m < k else 1.0)
        r = torch.sqrt(dx * dx + dy * dy)
        phi = (r * r) * torch.log(r + 1e-6)
        x = x + t[3 + m, 0] * phi
        y = y + t[3 + m, 1] * phi
    return x, y
