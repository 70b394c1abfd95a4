"""Text regions of full frames, without a GPU: the numpy restatement of the warp (region_warp_oracle.py) against live PIL
and the committed goldens, the size rule and the closed-form coefficients (parseq_b200/regions.py), the argument checks
of crop_regions, and the host-side checks of parseq_warp_regions on a NULL handle."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import make_golden_regions as mg
from parseq_b200.regions import box_quad, map_points, quad_coeffs, quad_size
from region_warp_oracle import pil_warp, warp


def test_restatement_equals_pil_on_seeded_cases():
    pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(7)
    n = 0
    while n < 200:
        frame, q = mg.random_case(rng)
        if not mg.convex(q):
            continue
        h, w = quad_size(q)
        a = quad_coeffs(q, h, w)
        assert np.array_equal(warp(frame, h, w, a), pil_warp(frame, h, w, a)), (n, q, frame.shape)
        n += 1


def test_goldens_regenerate_to_their_digests():
    frames, g = mg.load()
    quads = g["quads"].numpy()
    assert len(g["sha256"]) == len(quads) == len(g["frame_index"]) == len(g["sizes"])
    for i, (q, f, (h, w), a) in enumerate(zip(quads, g["frame_index"], g["sizes"], g["coeffs"].numpy())):
        assert mg.digest(warp(frames[f], h, w, a)) == g["sha256"][i], i


def test_golden_coefficients_and_sizes_are_the_closed_form_bit_for_bit():
    _, g = mg.load()
    for q, (h, w), a in zip(g["quads"].tolist(), g["sizes"], g["coeffs"].numpy()):
        assert quad_size(q) == (h, w)
        assert np.array_equal(np.array(quad_coeffs(q, h, w), dtype=np.float64).view(np.uint64), a.view(np.uint64)), q


def test_goldens_cover_the_edge_cases():
    _, g = mg.load()
    sizes = set(map(tuple, g["sizes"]))
    assert (1, 1) in sizes and any(h == 1 and w > 1 for h, w in sizes) and any(w == 8192 for _, w in sizes)
    assert {(1, 1), (4000, 6000)} <= {f[:2] for f in g["frames"]}
    idx = g["frame_index"]
    assert any(a != b for a, b in zip(idx, idx[1:])) and len(set(idx)) == len(g["frames"])


@pytest.mark.parametrize("box", [(37, 21, 137, 61), (0, 0, 1, 1), (-5, -3, 12, 9), (300, 230, 330, 250),
                                 (400, 300, 410, 305)])
def test_integer_boxes_are_pil_crops(box):
    Image = pytest.importorskip("PIL.Image")
    frame = mg.make_frame(240, 320, 9, 1)
    q = box_quad(box)
    h, w = quad_size(q)
    assert (h, w) == (box[3] - box[1], box[2] - box[0])
    a = quad_coeffs(q, h, w)
    assert a == (1.0, 0.0, float(box[0]), 0.0, 1.0, float(box[1]), 0.0, 0.0)
    assert np.array_equal(warp(frame, h, w, a), np.asarray(Image.fromarray(frame).crop(box)))


def test_integer_corner_quad_is_a_translation():
    q = [(37.0, 21.0), (137.0, 21.0), (137.0, 61.0), (37.0, 61.0)]
    assert quad_coeffs(q, *quad_size(q)) == (1.0, 0.0, 37.0, 0.0, 1.0, 21.0, 0.0, 0.0)


def test_map_sends_crop_corners_to_quad_corners():
    _, g = mg.load()
    rng = np.random.default_rng(3)
    quads = g["quads"].tolist() + [mg.random_case(rng)[1] for _ in range(100)]
    for q in quads:
        if not mg.convex(q):
            continue
        h, w = quad_size(q)
        a = quad_coeffs(q, h, w)
        scale = max(1.0, max(abs(v) for p in q for v in p))
        for (u, v), (x, y) in zip(((0, 0), (w, 0), (w, h), (0, h)), q):
            mx, my = map_points(a, float(u), float(v))
            assert abs(mx - x) <= 1e-9 * scale and abs(my - y) <= 1e-9 * scale, (q, u, v)


def test_size_rule():
    # the longer of the two opposite sides, rounded half up, at least 1
    assert quad_size([(0, 0), (10.4, 0), (10.4, 3), (0, 3)]) == (3, 10)
    assert quad_size([(0, 0), (10.5, 0), (10.5, 2.5), (0, 2.5)]) == (3, 11)
    assert quad_size([(0, 0), (9, 0), (12, 4), (0, 4)]) == (5, 12)          # |BR - TR| = 5, |BR - BL| = 12
    assert quad_size([(0, 0), (0.3, 0), (0.3, 0.3), (0, 0.3)]) == (1, 1)
    assert quad_size([(0, 0), (30, 40), (26, 43), (-4, 3)]) == (5, 50)     # a turned 50 x 5
    c, s = math.cos(1.0), math.sin(1.0)
    q = mg.rect(0.0, 0.0, 100, 20, c, s)
    assert quad_size(q) == (20, 100)


# ---------------------------------------------------------------- crop_regions argument checks
@pytest.fixture(scope="module")
def model():
    from parseq_b200.factory import create_model
    return create_model("parseq-tiny")


FRAME = torch.zeros((40, 60, 3), dtype=torch.uint8)
OK = [[[1.0, 1.0], [20.0, 2.0], [20.0, 12.0], [1.0, 11.0]]]


@pytest.mark.parametrize("regions, kw, msg", [
    ([[[1.0, 1.0], [math.inf, 2.0], [20.0, 12.0], [1.0, 11.0]]], {}, "non-finite"),
    ([[[1.0, 1.0], [math.nan, 2.0], [20.0, 12.0], [1.0, 11.0]]], {}, "non-finite"),
    ([[[5.0, 5.0], [5.0, 5.0], [5.0, 5.0], [5.0, 5.0]]], {}, "degenerate"),
    ([[[0.0, 0.0], [10.0, 0.0], [20.0, 0.0], [30.0, 0.0]]], {}, "degenerate"),
    ([[[0.0, 0.0], [10.0, 0.0], [0.0, 10.0], [10.0, 10.0]]], {}, "self-intersecting"),
    ([[[0.0, 0.0], [10.0, 0.0], [3.0, 3.0], [0.0, 10.0]]], {}, "not convex"),
    ([[[0.0, 0.0], [8193.0, 0.0], [8193.0, 5.0], [0.0, 5.0]]], {}, "at most 8192"),
    ([[0, 0, 8193, 4]], {}, "at most 8192"),
    ([[[0.0, 0.0], [1.0, 0.0], [1.0, 1.0]]], {}, "shape"),
    ([[0.0, 0.0, 1.0, 1.0, 2.0]], {}, "shape"),
    ([[1.0, 1.0], [2.0, 2.0], [2.0, 1.0], [1.0, 2.0]], {}, "shape"),
    (np.zeros((0, 4, 2)), {}, "M >= 1"),
    ([[1.5, 2.0, 10.0, 12.0]], {}, "integers"),
    ([[10, 2, 5, 12]], {}, "x1 > x0"),
    ([[0, 12, 5, 12]], {}, "x1 > x0"),
    (np.ones((1, 4, 2), dtype=bool), {}, "dtype"),
    (OK, {"frame_index": [1]}, "frame_index must be in"),
    (OK, {"frame_index": [-1]}, "frame_index must be in"),
    (OK, {"frame_index": [0, 0]}, "frame_index must be integer"),
    (OK, {"frame_index": [0.0]}, "frame_index must be integer"),
], ids=["inf", "nan", "point", "collinear", "bow_tie", "dart", "side_8193", "box_8193", "three_corners", "five_values",
        "one_quad_no_batch", "empty", "float_box", "box_x_reversed", "box_empty_y", "bool", "index_past", "index_negative",
        "index_length", "index_float"])
def test_crop_regions_rejects(model, regions, kw, msg):
    with pytest.raises(ValueError, match=msg):
        model.crop_regions(FRAME, regions, **kw)


def test_crop_regions_takes_tensors_and_arrays_alike(model):
    with pytest.raises(ValueError, match="self-intersecting"):
        model.crop_regions(FRAME, torch.tensor([[[0.0, 0.0], [10.0, 0.0], [0.0, 10.0], [10.0, 10.0]]]))
    with pytest.raises(ValueError, match="x1 > x0"):
        model.crop_regions(FRAME, torch.tensor([[10, 2, 5, 12]], dtype=torch.int32))


def test_crop_regions_rejects_bad_frames(model):
    with pytest.raises(ValueError, match="frame_index is required"):
        model.crop_regions([FRAME, FRAME], OK)
    with pytest.raises(ValueError, match="frame 0"):
        model.crop_regions(FRAME.float(), OK)
    with pytest.raises(ValueError, match="frame 1"):
        model.crop_regions([FRAME, FRAME[..., :2]], OK, frame_index=[1])
    with pytest.raises(ValueError, match="no frames"):
        model.crop_regions([], OK)
    Image = pytest.importorskip("PIL.Image")
    with pytest.raises(ValueError, match="mode RGB"):
        model.crop_regions(Image.new("L", (60, 40)), OK)


def test_region_crops_to_frame_and_packing():
    from parseq_b200.system import RegionCrops, pack_crops
    data = torch.arange(3 * 2 * 2 + 3 * 1 * 3, dtype=torch.uint8)
    views = [data[:12].view(2, 2, 3), data[12:].view(1, 3, 3)]
    q = [box_quad((5, 7, 7, 9)), [(0.0, 0.0), (3.0, 0.5), (3.0, 1.5), (0.0, 1.0)]]
    sizes = [quad_size(x) for x in q]
    cf = torch.tensor([quad_coeffs(x, *s) for x, s in zip(q, sizes)], dtype=torch.float64)
    rc = RegionCrops(views, data, torch.tensor([0, 12]), torch.tensor(sizes, dtype=torch.int32),
                     torch.tensor(q, dtype=torch.float64), cf, torch.tensor([0, 0]))
    assert isinstance(rc, list) and len(rc) == 2
    d, o, s = pack_crops(rc)
    assert d is data and o.tolist() == [0, 12] and s.tolist() == [[2, 2], [1, 3]]
    assert torch.equal(rc.to_frame([[0.0, 0.0], [2.0, 2.0], [0.5, 1.5]], 0),
                       torch.tensor([[5.0, 7.0], [7.0, 9.0], [5.5, 8.5]], dtype=torch.float64))
    h, w = sizes[1]
    corners = rc.to_frame(torch.tensor([[0.0, 0.0], [w, 0.0], [w, h], [0.0, h]]), 1)
    assert torch.allclose(corners, torch.tensor(q[1], dtype=torch.float64), rtol=0, atol=1e-12)
    rc.append(views[0])                       # no longer the packed list: packed like any other list
    d2, o2, _ = pack_crops(rc)
    assert d2 is not data and o2.tolist() == [0, 12, 21]


# ---------------------------------------------------------------- C ABI, host-side checks
@pytest.fixture(scope="module")
def lib():
    from parseq_b200.engine import load_library
    try:
        return load_library()
    except (RuntimeError, OSError) as e:
        pytest.skip(str(e))


def _regions(frame_sizes=((40, 60),), frames_bytes=None, frame_offsets=None, index=(0,), sizes=((10, 20),),
             coeffs=None, num_frames=None):
    from parseq_b200.engine import RegionsC
    fs = np.asarray(frame_sizes, dtype=np.int32).reshape(-1, 2)
    nb = 3 * fs[:, 0].astype(np.int64) * fs[:, 1]
    fo = np.asarray(frame_offsets, dtype=np.int64) if frame_offsets is not None else np.concatenate([[0], np.cumsum(nb)[:-1]])
    fi = np.asarray(index, dtype=np.int32)
    sz = np.asarray(sizes, dtype=np.int32).reshape(-1, 2)
    cf = (np.asarray(coeffs, dtype=np.float64).reshape(-1, 8) if coeffs is not None
          else np.tile(np.array([1, 0, 2, 0, 1, 3, 0, 0], dtype=np.float64), (len(fi), 1)))
    buf = np.zeros(16, dtype=np.uint8)         # never read: every check runs before the handle's
    r = RegionsC(buf.ctypes.data, int(nb.sum()) if frames_bytes is None else frames_bytes, fo.ctypes.data, fs.ctypes.data,
                 len(fs) if num_frames is None else num_frames, fi.ctypes.data, sz.ctypes.data, cf.ctypes.data)
    return r, (buf, fs, fo, fi, sz, cf)


def _warp(lib, r, count=1, out_bytes=1 << 20, out=True):
    o = (C.c_uint8 * 16)()
    return lib.parseq_warp_regions(None, count, C.byref(r) if r is not None else None, o if out else None, out_bytes, None)


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
    ({"coeffs": [1, 0, 2, 0, math.inf, 3, 0, 0]}, {}, "non-finite"),
    ({"coeffs": [1, 0, 2, 0, 1, math.nan, 0, 0]}, {}, "non-finite"),
    ({"coeffs": [1, 0, 2, 0, 1, 3, -0.2, 0]}, {}, "not positive"),        # 1 - 0.2 * 19.5 < 0 at the right corners
    ({"coeffs": [1, 0, 2, 0, 1, 3, 0, -2.0]}, {}, "not positive"),       # exactly 0 at the top corners (y + .5 = .5)
    ({}, {"out_bytes": 599}, "smaller than the packed crops"),
    ({}, {"count": -1}, "negative count"),
    ({}, {"out": False}, "null"),
], ids=["frame_side_0", "frame_side_32769", "frame_past_bytes", "frame_negative_offset", "no_frames", "index_past",
        "index_negative", "size_0", "size_8193", "coeff_inf", "coeff_nan", "denominator_negative", "denominator_zero",
        "out_bytes", "negative_count", "null_out"])
def test_warp_regions_rejects_without_a_device(lib, kw, call, msg):
    r, keep = _regions(**kw)
    assert _warp(lib, r, **call) < 0
    assert msg in lib.parseq_last_error().decode()


def test_warp_regions_rejects_null_pointers(lib):
    from parseq_b200.engine import RegionsC
    assert _warp(lib, None) < 0
    assert "null argument" in lib.parseq_last_error().decode()
    for field in ("frames", "frame_offsets", "frame_sizes", "frame_index", "sizes", "coeffs"):
        r, keep = _regions()
        setattr(r, field, None)
        assert _warp(lib, r) < 0, field
        assert "null frames" in lib.parseq_last_error().decode()
    # valid metadata reaches the handle check
    r, keep = _regions(frame_sizes=((40, 60), (5, 5)), index=(1, 0), sizes=((10, 20), (1, 1)),
                       coeffs=[[1, 0, 2, 0, 1, 3, 0, 0], [0.5, 0, 0, 0, 0.5, 0, 1e-3, -2e-3]])
    assert _warp(lib, r, count=2, out_bytes=603) < 0
    assert "null argument" in lib.parseq_last_error().decode()
    assert RegionsC is not None
