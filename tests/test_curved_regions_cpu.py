"""Curved text regions without a GPU: parseq_tps_coeffs and the fp64 restatement (tps_warp_oracle.py) against the
reference's own thin-plate-spline grids (goldens of make_golden_curved.py), the fiducials and the size rule, the argument
checks of crop_regions for polygons, and the host-side checks of parseq_warp_polygons on a NULL handle."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import make_golden_curved as mgc
import make_golden_regions as mg
from parseq_b200.regions import check_polygon, engine_points, map_points, map_tps, polygon_size, quad_coeffs, quad_size
from tps_warp_oracle import sample, tps_map


@pytest.fixture(scope="module")
def lib():
    from parseq_b200.engine import load_library
    try:
        return load_library()
    except (RuntimeError, OSError) as e:
        pytest.skip(str(e))


@pytest.fixture(scope="module")
def golden():
    return mgc.load()


def _coeffs(lib, engine_pts):
    from parseq_b200.engine import tps_coeffs
    return tps_coeffs(engine_pts, lib)


def test_coefficients_and_oracle_map_equal_the_reference_grids(lib, golden):
    """Within 1e-11 of the polygon's coordinate scale: at most 1e-9 px for coordinates up to 100 px.  inv_delta_C is
    ill-conditioned enough at k = 32 that numpy's LAPACK inverse and the engine's Gauss-Jordan one part in 1e12."""
    _, g = golden
    worst = 0.0
    for p, (h, w), idx, ref in zip(g["polygons"], g["sizes"], g["samples"], g["mapped"]):
        t = _coeffs(lib, engine_points(p.tolist()))
        scale = max(100.0, float(p.abs().max()))
        X, Y = tps_map(t, h, w)
        got = np.stack([X.reshape(-1), Y.reshape(-1)], -1)[idx.numpy()]
        err = float(np.abs(got - ref.numpy()).max())
        assert err <= 1e-11 * scale, (err, scale)
        worst = max(worst, err / scale)
        # to_frame's map at the pixel centres is the same map, up to the rounding of xn = 2u / w - 1
        yy, xx = np.divmod(idx.numpy(), w)
        mx, my = map_tps(t, h, w, torch.from_numpy(xx + 0.5), torch.from_numpy(yy + 0.5))
        assert float((torch.stack([mx, my], -1) - ref).abs().max()) <= 1e-11 * scale
    print(f"largest distance to the reference grids: {worst:.3g} of the coordinate scale")


def test_sampler_tail_equals_the_quad_restatement_on_its_goldens():
    """tps_warp_oracle.sample at the perspective map's points makes region_warp_oracle.warp's bytes, which equal PIL's
    (test_regions_cpu.py), on every quad golden and on seeded quads."""
    from region_warp_oracle import warp
    frames, g = mg.load()
    cases = [(frames[f], h, w, a) for f, (h, w), a in zip(g["frame_index"], g["sizes"], g["coeffs"].numpy())]
    rng = np.random.default_rng(5)
    while len(cases) < len(g["sizes"]) + 50:
        frame, q = mg.random_case(rng)
        if mg.convex(q):
            h, w = quad_size(q)
            cases.append((frame, h, w, quad_coeffs(q, h, w)))
    for frame, h, w, a in cases:
        a0, a1, a2, a3, a4, a5, a6, a7 = (float(c) for c in a)
        yin, xin = np.meshgrid(np.arange(h, dtype=np.float64) + 0.5, np.arange(w, dtype=np.float64) + 0.5, indexing="ij")
        den = a6 * xin + a7 * yin + 1.0
        sx, sy = (a0 * xin + a1 * yin + a2) / den, (a3 * xin + a4 * yin + a5) / den
        assert np.array_equal(sample(frame, sx, sy), warp(frame, h, w, a)), (frame.shape, h, w)


def test_fiducial_x_is_numpy_linspace_bit_for_bit(lib):
    # an affine polygon with top y = 0 and unit spacing: the coefficients then hold nothing of C_x, so test C_x
    # through the restatement the kernel follows (j * (2 / (k - 1)) + (-1), last point 1)
    for k in range(3, 33):
        step = 2.0 / (k - 1)
        cx = np.array([j * step + (-1.0) for j in range(k - 1)] + [1.0])
        assert np.array_equal(cx.view(np.uint64), np.linspace(-1.0, 1.0, k).view(np.uint64)), k


def test_size_rule_reduces_to_quad_size_and_reverses_the_bottom_edge():
    rng = np.random.default_rng(11)
    for _ in range(200):
        _, q = mg.random_case(rng)
        # a quad as the two-point edges p = (TL, TR), b = (BL, BR): the engine order of caller order TL, TR, BR, BL
        assert polygon_size(engine_points(q)) == quad_size(q)
    poly = [(0.0, 0.0), (10.0, 0.0), (20.0, 0.0), (20.0, 5.0), (10.0, 6.0), (0.0, 7.0)]
    assert engine_points(poly) == [(0.0, 0.0), (10.0, 0.0), (20.0, 0.0), (0.0, 7.0), (10.0, 6.0), (20.0, 5.0)]
    assert polygon_size(engine_points(poly)) == (7, 20)


def test_affine_polygon_maps_like_its_quad(lib):
    for cx, cy, w, h, a, k in ((160.3, 120.7, 140, 32, 0.4, 7), (200.0, 150.0, 90, 24, 0.0, 16), (3000.5, 2000.25, 640, 96, -1.1, 32),
                               (12.0, 7.0, 20, 3, 2.0, 3)):
        p = mgc.affine_polygon(cx, cy, w, h, a, k)
        kk = len(p) // 2
        quad = [p[0], p[kk - 1], p[kk], p[-1]]
        hh, ww = polygon_size(engine_points(p))
        assert (hh, ww) == quad_size(quad)
        X, Y = tps_map(_coeffs(lib, engine_points(p)), hh, ww)
        yy, xx = np.meshgrid(np.arange(hh) + 0.5, np.arange(ww) + 0.5, indexing="ij")
        qx, qy = map_points(quad_coeffs(quad, hh, ww), xx, yy)
        scale = max(100.0, max(abs(v) for pt in p for v in pt))     # 1e-9 px up to 100 px, as above
        assert max(float(np.abs(X - qx).max()), float(np.abs(Y - qy).max())) <= 1e-11 * scale, (cx, cy, k)


@pytest.mark.skipif(not mgc.reference_available(), reason="the reference tree is not present")
def test_goldens_regenerate():
    _, g = mgc.load()
    new = mgc.build(mgc.grid_generator())
    assert new["frame_index"] == g["frame_index"] and new["sizes"] == g["sizes"]
    for a, b in zip(new["polygons"], g["polygons"]):
        assert torch.equal(a, b)
    for a, b in zip(new["samples"], g["samples"]):
        assert torch.equal(a, b)
    for a, b in zip(new["mapped"], g["mapped"]):      # LAPACK builds may differ in the last bits of inv_delta_C
        assert float((a - b).abs().max()) <= 1e-9


def test_goldens_cover_the_edge_cases(golden):
    _, g = golden
    ks = {len(p) // 2 for p in g["polygons"]}
    assert {3, 7, 16, 32} <= ks
    sizes = set(map(tuple, g["sizes"]))
    assert any(h == 1 and w > 1 for h, w in sizes) and any(w == 8192 for _, w in sizes) and (1, 1) in sizes
    assert {2, 3} <= set(g["frame_index"])


# ---------------------------------------------------------------- crop_regions argument checks
@pytest.fixture(scope="module")
def model():
    from parseq_b200.factory import create_model
    return create_model("parseq-tiny")


FRAME = torch.zeros((40, 60, 3), dtype=torch.uint8)
ARC = [(1.0, 5.0), (10.0, 2.0), (20.0, 5.0), (18.0, 12.0), (10.0, 9.0), (3.0, 12.0)]


@pytest.mark.parametrize("regions, msg", [
    ([ARC[:5]], "region 0: 5 points"),
    ([ARC + [(0.0, 8.0)]], "region 0: 7 points"),
    ([ARC, ARC[:5]], "region 1: 5 points"),
    ([ARC, [(0.0, 0.0), (1.0, 0.0)]], "region 1: 2 points"),
    ([ARC, [(0.0, 0.0)] * 66], "region 1: 66 points"),
    ([[(float(j), 0.0) for j in range(33)] + [(float(j), 5.0) for j in range(33)][::-1]], "region 0: 66 points"),
    ([ARC[:2] + [(math.inf, 5.0)] + ARC[3:]], "region 0: non-finite"),
    ([[[1.0, 1.0], [20.0, 2.0], [20.0, 12.0], [1.0, 11.0]], ARC[:2] + [(math.nan, 5.0)] + ARC[3:]], "region 1: non-finite"),
    ([[(0.0, 0.0), (10.0, 0.0), (20.0, 0.0), (0.0, 10.0), (10.0, 10.0), (20.0, 10.0)]], "region 0: the polygon is self-intersecting"),
    ([[(0.0, 0.0), (10.0, 12.0), (20.0, 0.0), (20.0, 10.0), (10.0, 5.0), (0.0, 10.0)]], "region 0: the polygon is self-intersecting"),
    ([[(0.0, 0.0), (10.0, 0.0), (5.0, 0.0), (5.0, 10.0), (10.0, 10.0), (0.0, 10.0)]], "region 0: the polygon is self-intersecting"),
    ([[(0.0, 0.0), (10.0, 0.0), (10.0, 0.0), (20.0, 10.0), (10.0, 10.0), (0.0, 10.0)]], "region 0: the polygon is degenerate"),
    ([[(0.0, 0.0), (4100.0, 0.0), (8200.0, 0.0), (8200.0, 5.0), (4100.0, 5.0), (0.0, 5.0)]], "region 0: crop size 5 x 8200"),
    ([[(0.0, 0.0), (5.0, 0.0), (10.0, 0.0), (10.0, 8200.0), (5.0, 8200.0), (0.0, 8200.0)]], "region 0: crop size 8200"),
    ([ARC, np.zeros((6, 3))], "region 1: points must be real"),
], ids=["five", "seven", "ragged_five", "ragged_two", "ragged_66", "sixty_six", "inf", "nan_after_quad", "bow_tie",
        "crossing_edges", "fold_back", "repeated_point", "width_8200", "height_8200", "bad_shape"])
def test_crop_regions_rejects_polygons(model, regions, msg):
    with pytest.raises(ValueError, match=msg.replace("(", r"\(")):
        model.crop_regions(FRAME, regions)


def test_check_polygon_accepts_the_goldens_and_both_windings(golden):
    _, g = golden
    for i, p in enumerate(g["polygons"]):
        check_polygon(p.tolist(), i)
    check_polygon(ARC)
    check_polygon(ARC[::-1])


def test_region_crops_to_frame_of_a_polygon(lib):
    from parseq_b200.system import RegionCrops
    p = mgc.band(mgc.arc(160.0, 200.0, 120.0, -150.0, -30.0), 7, 14.0)
    e = engine_points(p)
    h, w = polygon_size(e)
    t = torch.from_numpy(_coeffs(lib, e))
    data = torch.zeros(3 * h * w, dtype=torch.uint8)
    rc = RegionCrops([data.view(h, w, 3)], data, torch.tensor([0]), torch.tensor([[h, w]], dtype=torch.int32),
                     torch.tensor([[p[0], p[6], p[7], p[-1]]], dtype=torch.float64), torch.full((1, 8), math.nan,
                                                                                          dtype=torch.float64),
                     torch.tensor([0]), [torch.tensor(p, dtype=torch.float64)], [t])
    corners = rc.to_frame(torch.tensor([[0.0, 0.0], [w, 0.0], [w, h], [0.0, h]], dtype=torch.float64), 0)
    # the corners are fiducials, where phi uses ln(r + 1e-6) rather than the solve's ln r (GridGenerator's own map
    # misses them by as much): within 1e-4 px
    assert float((corners - rc.quads[0]).abs().max()) <= 1e-4


# ---------------------------------------------------------------- C ABI, host-side checks
def test_tps_coeffs_rejects(lib):
    pts = np.zeros((6, 2))
    out = np.zeros((9, 2))
    for n, msg in ((5, "even count"), (4, "even count"), (66, "even count")):
        assert lib.parseq_tps_coeffs(n, pts.ctypes.data, out.ctypes.data) < 0
        assert msg in lib.parseq_last_error().decode()
    assert lib.parseq_tps_coeffs(6, None, out.ctypes.data) < 0
    assert "null" in lib.parseq_last_error().decode()
    bad = pts.copy()
    bad[3, 1] = math.nan
    assert lib.parseq_tps_coeffs(6, bad.ctypes.data, out.ctypes.data) < 0
    assert "non-finite" in lib.parseq_last_error().decode()


def _polygons(frame_sizes=((40, 60),), frames_bytes=None, frame_offsets=None, index=(0,), sizes=((10, 20),),
              num_points=(6,), points=None, num_frames=None):
    from parseq_b200.engine import PolygonsC
    fs = np.asarray(frame_sizes, dtype=np.int32).reshape(-1, 2)
    nb = 3 * fs[:, 0].astype(np.int64) * fs[:, 1]
    fo = np.asarray(frame_offsets, dtype=np.int64) if frame_offsets is not None else np.concatenate([[0], np.cumsum(nb)[:-1]])
    fi = np.asarray(index, dtype=np.int32)
    sz = np.asarray(sizes, dtype=np.int32).reshape(-1, 2)
    npt = np.asarray(num_points, dtype=np.int32)
    pts = (np.asarray(points, dtype=np.float64).reshape(-1, 2) if points is not None
           else np.tile(np.array(engine_points(ARC), dtype=np.float64), (max(1, int(npt.sum()) // 6 + 1), 1)))
    buf = np.zeros(16, dtype=np.uint8)         # never read: every check runs before the handle's
    r = PolygonsC(buf.ctypes.data, int(nb.sum()) if frames_bytes is None else frames_bytes, fo.ctypes.data, fs.ctypes.data,
                  len(fs) if num_frames is None else num_frames, fi.ctypes.data, sz.ctypes.data, npt.ctypes.data,
                  pts.ctypes.data)
    return r, (buf, fs, fo, fi, sz, npt, pts)


def _warp(lib, r, count=1, out_bytes=1 << 20, out=True):
    o = (C.c_uint8 * 16)()
    return lib.parseq_warp_polygons(None, count, C.byref(r) if r is not None else None, o if out else None, out_bytes,
                                    None)


NAN_PTS = engine_points(ARC)[:3] + [(math.nan, 1.0)] + engine_points(ARC)[4:]


@pytest.mark.parametrize("kw, call, msg", [
    ({"frame_sizes": ((0, 60),)}, {}, "sides must be in [1, 32768]"),
    ({"frame_sizes": ((40, 32769),)}, {}, "sides must be in [1, 32768]"),
    ({"frames_bytes": 100}, {}, "exceeds frames_bytes"),
    ({"frame_offsets": [-3]}, {}, "exceeds frames_bytes"),
    ({"num_frames": 0}, {}, "num_frames"),
    ({"index": (1,)}, {}, "frame_index 1 out of range"),
    ({"index": (-1,)}, {}, "frame_index -1 out of range"),
    ({"sizes": ((0, 20),)}, {}, "sides must be in [1, 8192]"),
    ({"sizes": ((10, 8193),)}, {}, "sides must be in [1, 8192]"),
    ({"num_points": (7,)}, {}, "region 0: 7 points"),
    ({"num_points": (4,)}, {}, "region 0: 4 points"),
    ({"num_points": (66,)}, {}, "region 0: 66 points"),
    ({"points": NAN_PTS}, {}, "region 0: non-finite point"),
    ({"points": engine_points(ARC) + NAN_PTS, "num_points": (6, 6), "index": (0, 0), "sizes": ((4, 4), (4, 4))},
     {"count": 2}, "region 1: non-finite point"),
    ({}, {"out_bytes": 599}, "smaller than the packed crops"),
    ({}, {"count": -1}, "negative count"),
    ({}, {"out": False}, "null"),
], ids=["frame_side_0", "frame_side_32769", "frame_past_bytes", "frame_negative_offset", "no_frames", "index_past",
        "index_negative", "size_0", "size_8193", "odd_points", "four_points", "66_points", "nan_point",
        "nan_point_second_region", "out_bytes", "negative_count", "null_out"])
def test_warp_polygons_rejects_without_a_device(lib, kw, call, msg):
    r, keep = _polygons(**kw)
    assert _warp(lib, r, **call) < 0
    assert msg in lib.parseq_last_error().decode()


def test_warp_polygons_rejects_null_pointers(lib):
    assert _warp(lib, None) < 0
    assert "null argument" in lib.parseq_last_error().decode()
    for field in ("frames", "frame_offsets", "frame_sizes", "frame_index", "sizes", "num_points", "points"):
        r, keep = _polygons()
        setattr(r, field, None)
        assert _warp(lib, r) < 0, field
        assert "null frames" in lib.parseq_last_error().decode()
    # valid metadata, ragged k, reaches the handle check
    pts = engine_points(ARC) + [(float(j), 0.0) for j in range(8)] + [(float(j), 3.0) for j in range(8)]
    r, keep = _polygons(frame_sizes=((40, 60), (5, 5)), index=(1, 0), sizes=((10, 20), (1, 1)), num_points=(6, 16),
                        points=pts)
    assert _warp(lib, r, count=2, out_bytes=603) < 0
    assert "null argument" in lib.parseq_last_error().decode()
