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
