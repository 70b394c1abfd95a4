"""Writes tests/golden/curved/curved.pt: curved text regions (polygons of 2k points) on the seeded frames of
make_golden_regions.py, and the frame points the reference's own thin-plate spline gives their crop pixels.  Needs the
reference tree (oracle/reference_loader.py):

    python tests/make_golden_curved.py

The map is TRBA's GridGenerator (strhub/models/trba/transformation.py) with its numpy fp64 builders combined as
build_P_prime combines them: T = inv_delta_C . [C'; 0] and P' = P_hat . T, with C' the polygon in frame pixels (engine
order).  Only data is stored: per region its points (caller order: top edge left to right, bottom edge right to left),
frame index, crop size (h, w), a seeded sample of its pixel indices y * w + x (the four corners included) and P' at
them.  The polygons cover arcs of both curvatures, S-curves, circular sectors (CUTE80-like), vertical curved text,
polygons partly and wholly outside the frame, k = 3, 7 (CTW1500's 14 points), 16 and 32, an affine case (points evenly
spaced along the long sides of a turned rectangle), 1 x N and 8192-wide crops, the 1 x 1 frame and the 6000 x 4000
frame."""
from __future__ import annotations

import importlib.util
import math
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

import make_golden_regions as mg  # noqa: E402
from parseq_b200.regions import check_polygon, engine_points, polygon_size  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "curved", "curved.pt")
SAMPLES = 256                               # pixels per region whose reference map is stored (plus the corners)


def reference_path() -> str:
    from oracle import reference_loader
    return os.path.join(reference_loader.REF_ROOT, "strhub", "models", "trba", "transformation.py")


def reference_available() -> bool:
    return os.path.isfile(reference_path())


def grid_generator():
    """The reference's GridGenerator class, imported from its source file."""
    spec = importlib.util.spec_from_file_location("_ref_trba_transformation", reference_path())
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.GridGenerator


def reference_map(gg, points, h: int, w: int, idx) -> np.ndarray:
    """P' [len(idx), 2] of GridGenerator(F, (h, w)) at pixel indices idx for fiducials C' = points [F, 2] (engine
    order), in numpy fp64: the builders of __init__ and the two products of build_P_prime."""
    c_prime = np.asarray(points, dtype=np.float64)
    F = len(c_prime)
    me = types.SimpleNamespace(eps=1e-6)
    C = gg._build_C(me, F)
    inv_delta_C = gg._build_inv_delta_C(me, F, C)
    P = gg._build_P(me, w, h)
    P_hat = gg._build_P_hat(me, F, C, P[np.asarray(idx)])
    T = inv_delta_C @ np.concatenate([c_prime, np.zeros((3, 2))], axis=0)
    return P_hat @ T


def band(curve, k: int, half: float, s0: float = 0.0, s1: float = 1.0):
    """Polygon (caller order) of a text band of half-height `half` around the centre line curve(s), s0 <= s <= s1,
    read left to right; the normal (-t_y, t_x) of the unit tangent t points to the bottom edge."""
    top, bot = [], []
    for s in np.linspace(s0, s1, k):
        (xa, ya), (xb, yb) = curve(s - 1e-6), curve(s + 1e-6)
        tx, ty = xb - xa, yb - ya
        n = math.hypot(tx, ty)
        nx, ny = -ty / n, tx / n
        x, y = curve(s)
        top.append((x - half * nx, y - half * ny))
        bot.append((x + half * nx, y + half * ny))
    return top + bot[::-1]


def arc(cx, cy, r, a0, a1):
    """Centre line on a circle from angle a0 to a1 (degrees, y down): a0 < a1 runs over the top (a frown), a0 > a1
    under the bottom (a smile)."""
    return lambda s: (cx + r * math.cos(math.radians(a0 + (a1 - a0) * s)), cy + r * math.sin(math.radians(a0 + (a1 - a0) * s)))


def s_curve(x0, y0, length, amp, turns=1.0, angle=0.0):
    c, sn = math.cos(angle), math.sin(angle)

    def f(s):
        u, v = length * s, amp * math.sin(2 * math.pi * turns * s)
        return x0 + c * u - sn * v, y0 + sn * u + c * v
    return f


def line(x0, y0, x1, y1):
    return lambda s: (x0 + (x1 - x0) * s, y0 + (y1 - y0) * s)


def affine_polygon(cx, cy, w, h, angle, k):
    """A w x h rectangle turned by `angle`, k points evenly spaced along each long side (caller order)."""
    q = mg.rect(cx, cy, w, h, math.cos(angle), math.sin(angle))        # TL, TR, BR, BL
    top = [(q[0][0] + (q[1][0] - q[0][0]) * j / (k - 1), q[0][1] + (q[1][1] - q[0][1]) * j / (k - 1)) for j in range(k)]
    bot = [(q[3][0] + (q[2][0] - q[3][0]) * j / (k - 1), q[3][1] + (q[2][1] - q[3][1]) * j / (k - 1)) for j in range(k)]
    return top + bot[::-1]


def golden_polygons():
    """[(polygon in caller order, frame index)]."""
    out = [
        (band(arc(160.0, 200.0, 120.0, -150.0, -30.0), 7, 14.0), 0),            # frown, CTW1500's 14 points
        (band(arc(160.0, 20.0, 110.0, 150.0, 30.0), 7, 12.0), 0),               # smile
        (band(arc(210.0, 150.0, 90.0, -170.0, -10.0), 16, 16.0), 1),            # CUTE80-like sector, 160 degrees
        (band(arc(210.0, 150.0, 60.0, 200.0, -20.0), 32, 10.0), 1),             # under a logo, 220 degrees, k = 32
        (band(s_curve(20.0, 120.0, 280.0, 25.0), 16, 11.0), 0),                 # S-curve
        (band(s_curve(30.0, 60.0, 360.0, 18.0, 1.5, 0.3), 32, 9.5), 1),         # turned S-curve, 1.5 periods
        (band(s_curve(150.0, 20.0, 200.0, 20.0, 0.5, math.pi / 2), 7, 13.0), 0),  # vertical, read downwards
        (band(arc(260.0, 150.0, 100.0, -60.0, 60.0), 16, 12.0), 1),             # vertical arc on the right
        (band(arc(160.0, 200.0, 120.0, -150.0, -30.0), 3, 14.0), 0),            # k = 3
        (band(line(40.5, 60.25, 230.75, 90.5), 3, 8.0), 0),                     # k = 3, straight
        (affine_polygon(160.3, 120.7, 140, 32, 0.4, 7), 0),                     # affine
        (affine_polygon(200.0, 150.0, 90, 24, -1.1, 16), 1),                    # affine, k = 16
        (band(arc(-20.0, 40.0, 80.0, -120.0, 0.0), 7, 15.0), 0),                # partly outside
        (band(arc(900.0, 900.0, 80.0, -150.0, -30.0), 7, 15.0), 1),             # wholly outside
        (band(arc(60.0, 45.0, 300.0, -100.0, -80.0), 7, 0.3), 4),               # 1 x N
        (band(line(0.1, 0.5, 0.9, 0.5), 3, 0.3), 2),                            # the 1 x 1 frame: a 1 x 1 crop
        (band(arc(0.5, 6.0, 8.0, -135.0, -45.0), 7, 2.0), 2),                   # around the 1 x 1 frame
        (band(arc(3000.0, 2600.0, 900.0, -140.0, -40.0), 16, 48.0), 3),         # 6000 x 4000: a large arc
        (band(line(-1096.0, 2000.0, 7095.9, 2003.0), 32, 1.2), 3),              # 8192 wide, past both sides
        (band(arc(5000.0, 600.0, 500.0, 160.0, 20.0), 7, 30.0), 3),
    ]
    rng = np.random.default_rng(2025)
    while len(out) < 30:                                                       # seeded arcs of any k, turn and curvature
        f = len(out) % 2
        H, W = mg.FRAMES[f][:2]
        k = int(rng.choice([3, 4, 5, 7, 9, 12, 16, 24, 32]))
        a0 = rng.uniform(-170, -10)
        span = rng.uniform(10, 120) * rng.choice([-1, 1])
        r = rng.uniform(40, 300)
        poly = band(arc(rng.uniform(0, W), rng.uniform(0, H) + r, r, a0, a0 + span), k, rng.uniform(4, 20))
        try:
            check_polygon(poly)
        except ValueError:
            continue
        out.append((poly, f))
    for i, (p, _) in enumerate(out):
        check_polygon(p, i)
    return out


def sample_index(h: int, w: int, seed: int) -> np.ndarray:
    n = h * w
    corners = np.array([0, w - 1, (h - 1) * w, n - 1], dtype=np.int64)
    rng = np.random.default_rng(seed)
    pick = rng.choice(n, size=min(n, SAMPLES), replace=False) if n > 0 else np.zeros(0, dtype=np.int64)
    return np.unique(np.concatenate([corners, pick.astype(np.int64)]))


def build(gg):
    """The golden dict, from the reference's GridGenerator class."""
    import torch
    fs = mg.frames()
    polys = golden_polygons()
    sizes, index, samples, mapped = [], [], [], []
    for i, (p, f) in enumerate(polys):
        e = engine_points(p)
        h, w = polygon_size(e)
        idx = sample_index(h, w, 1000 + i)
        sizes.append((h, w))
        index.append(f)
        samples.append(torch.from_numpy(idx))
        mapped.append(torch.from_numpy(reference_map(gg, e, h, w, idx)))
    return {"frames": mg.FRAMES, "frame_sha256": [mg.digest(x) for x in fs],
            "polygons": [torch.tensor(p, dtype=torch.float64) for p, _ in polys], "frame_index": index,
            "sizes": sizes, "samples": samples, "mapped": mapped}


def load():
    """(frames, golden dict), the frames checked against their recorded digests."""
    import torch
    g = torch.load(OUT, weights_only=False)
    fs = mg.frames()
    assert [mg.digest(f) for f in fs] == g["frame_sha256"], "the golden frames do not regenerate to the recorded bytes"
    return fs, g


def main():
    import torch
    g = build(grid_generator())
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    torch.save(g, OUT)
    print(OUT, len(g["polygons"]), "regions", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
