"""Writes tests/golden/regions/regions.pt: text regions of seeded frames and the SHA-256 digest of what PIL makes of each,
frame.transform((w, h), PERSPECTIVE, coeffs, BICUBIC).  Needs PIL:

    python tests/make_golden_regions.py

The frames are regenerated, not stored: splitmix64 of the byte index (oracle/make_golden_crops.py `pixels`), either per
pixel ("noise") or per cell of `cell` x `cell` pixels ("blocky", so that the bicubic taps also see flat areas and
edges).  The file holds each frame's spec and digest, and per region its quad (TL, TR, BR, BL), frame index, size (h, w),
coefficient doubles (parseq_b200/regions.py) and output digest.  The regions cover rotated rectangles at many angles
(exact multiples of 90 degrees and 1e-9 degrees either side of them), perspective quads with strong foreshortening (one
axis minified), integer boxes, regions partly and wholly outside their frame, 1 x 1 and 1 x N crops, an 8192-wide crop,
a 1 x 1 frame and a 6000 x 4000 frame, with the frame indices interleaved."""
from __future__ import annotations

import hashlib
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.make_golden_crops import pixels  # noqa: E402
from parseq_b200.regions import box_quad, check_quad, quad_coeffs, quad_size  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "regions", "regions.pt")

# (H, W, seed, cell): cell 1 = noise
FRAMES = [(240, 320, 101, 1), (300, 420, 102, 6), (1, 1, 103, 1), (4000, 6000, 104, 16), (90, 700, 105, 3)]


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def make_frame(H: int, W: int, seed: int, cell: int) -> np.ndarray:
    if cell == 1:
        return pixels(H, W, seed)
    small = pixels((H + cell - 1) // cell, (W + cell - 1) // cell, seed)
    return np.repeat(np.repeat(small, cell, 0), cell, 1)[:H, :W]


def frames():
    return [make_frame(*f) for f in FRAMES]


def rect(cx, cy, w, h, c, s):
    """The quad of a w x h rectangle centred at (cx, cy), turned by the rotation (c, s) = (cos, sin)."""
    return [(cx + c * x - s * y, cy + s * x + c * y) for x, y in ((-w / 2, -h / 2), (w / 2, -h / 2), (w / 2, h / 2),
                                                                  (-w / 2, h / 2))]


def perspective(rng, cx, cy, w, h, jitter):
    """A turned rectangle with each corner moved by up to jitter * its size."""
    th = rng.uniform(-math.pi / 4, math.pi / 4)
    q = rect(cx, cy, w, h, math.cos(th), math.sin(th))
    return [(x + rng.uniform(-jitter, jitter) * w, y + rng.uniform(-jitter, jitter) * h) for x, y in q]


def convex(q) -> bool:
    try:
        check_quad(q)
    except ValueError:
        return False
    return True


def golden_regions():
    """[(quad, frame index)] of the golden file."""
    out = []
    exact = {0: (1.0, 0.0), 90: (0.0, 1.0), 180: (-1.0, 0.0), 270: (0.0, -1.0)}
    angles = [0, 90, 180, 270, 0.5, 15, 30, 45, 60, 89, 135, 200, 300, -30, -89.9]
    for k, a in enumerate(angles):
        c, s = exact.get(a, (math.cos(math.radians(a)), math.sin(math.radians(a))))
        out.append((rect(160.3, 120.7, 120, 30, c, s), k % 2))
    for a in (0, 90, 180, 270):
        for eps in (-1e-9, 1e-9):
            r = math.radians(a + eps)
            out.append((rect(200.0, 150.0, 90, 24, math.cos(r), math.sin(r)), 1))
    # strong foreshortening: the far side a fraction of the near one, so that side's axis minifies
    out.append(([(10.0, 20.0), (300.0, 95.0), (300.0, 110.0), (10.0, 200.0)], 0))
    out.append(([(40.0, 40.0), (380.0, 10.0), (360.0, 290.0), (60.0, 160.0)], 1))
    out.append(([(5.5, 60.25), (690.0, 10.0), (690.0, 80.0), (5.5, 70.0)], 4))
    rng = np.random.default_rng(2024)
    while len(out) < len(angles) + 8 + 3 + 12:
        f = len(out) % 2
        H, W = FRAMES[f][:2]
        q = perspective(rng, rng.uniform(0, W), rng.uniform(0, H), rng.uniform(30, 250), rng.uniform(10, 60), 0.15)
        if convex(q):
            out.append((q, f))
    # integer boxes: inside, partly outside, wholly outside
    for box, f in (((37, 21, 137, 61), 0), ((300, 200, 400, 260), 0), ((-20, -5, 30, 17), 1), ((500, 400, 540, 420), 1),
                   ((0, 0, 1, 1), 2), ((-3, -2, 4, 2), 2)):
        out.append((box_quad(box), f))
    # partly and wholly outside
    out.append((rect(-10.0, 5.0, 80, 30, math.cos(0.3), math.sin(0.3)), 0))
    out.append((rect(1000.0, 1000.0, 60, 20, math.cos(0.1), math.sin(0.1)), 1))
    # 1 x 1 and 1 x N crops; around the 1 x 1 frame
    out.append(([(5.0, 5.0), (5.4, 5.1), (5.3, 5.4), (4.9, 5.3)], 0))
    out.append(([(10.0, 50.0), (210.0, 53.0), (210.0, 53.3), (10.0, 50.3)], 1))
    out.append(([(0.1, 0.2), (0.9, 0.1), (0.8, 0.9), (0.2, 0.8)], 2))
    out.append((rect(0.5, 0.5, 12, 5, math.cos(0.7), math.sin(0.7)), 2))
    # the 6000 x 4000 frame: ordinary words, an 8192-wide crop that runs past both sides, a steep perspective quad
    out.append((rect(3000.0, 2000.0, 640, 96, math.cos(0.2), math.sin(0.2)), 3))
    out.append(([(-1096.0, 1500.0), (7096.0, 1502.0), (7096.0, 1505.0), (-1096.0, 1503.0)], 3))
    out.append(([(100.0, 3900.0), (5900.0, 100.0), (5950.0, 250.0), (150.0, 3990.0)], 3))
    return out


def random_case(rng):
    """(frame, quad) of the generator's distribution for the live PIL comparison: a noise or blocky frame of up to
    300 x 400, a rectangle of 1-200 x 1-60 at any angle with up to 10 % perspective, centred up to 20 px outside."""
    H, W = int(rng.integers(1, 300)), int(rng.integers(1, 400))
    frame = make_frame(H, W, int(rng.integers(1, 1 << 30)), int(rng.choice([1, 1, 5, 9])))
    th = rng.uniform(-math.pi, math.pi)
    q = rect(rng.uniform(-20, W + 20), rng.uniform(-20, H + 20), rng.uniform(1, 200), rng.uniform(1, 60), math.cos(th),
             math.sin(th))
    if rng.uniform() < 0.5:
        d = 0.1 * min(abs(q[1][0] - q[0][0]) + abs(q[1][1] - q[0][1]), abs(q[3][0] - q[0][0]) + abs(q[3][1] - q[0][1]))
        q = [(x + rng.uniform(-d, d), y + rng.uniform(-d, d)) for x, y in q]
    return frame, q


def load():
    """(frames, golden dict), the frames checked against their recorded digests."""
    import torch
    g = torch.load(OUT, weights_only=False)
    fs = frames()
    assert [digest(f) for f in fs] == g["frame_sha256"], "the golden frames do not regenerate to the recorded bytes"
    return fs, g


def main():
    import torch
    from region_warp_oracle import pil_warp
    fs = frames()
    regions = golden_regions()
    quads = np.array([q for q, _ in regions], dtype=np.float64)
    sizes = [quad_size(q) for q, _ in regions]
    coeffs = np.array([quad_coeffs(q, h, w) for (q, _), (h, w) in zip(regions, sizes)], dtype=np.float64)
    index = [f for _, f in regions]
    outs = [pil_warp(fs[f], h, w, a) for f, (h, w), a in zip(index, sizes, coeffs)]
    g = {"frames": FRAMES, "frame_sha256": [digest(f) for f in fs], "quads": torch.from_numpy(quads),
         "frame_index": index, "sizes": sizes, "coeffs": torch.from_numpy(coeffs),
         "sha256": [digest(o) for o in outs]}
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    torch.save(g, OUT)
    print(OUT, len(regions), "regions", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    main()
