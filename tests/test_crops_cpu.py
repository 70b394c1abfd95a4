"""Raw crops of any size, without a GPU: the numpy oracle of the engine's resize (oracle/crop_transform.py) against live
PIL / torchvision and the committed goldens of the reference's own transform, the Python packing of crop lists, and the
host-side checks of the crop entry points of the C ABI."""
import ctypes as C

import numpy as np
import pytest
import torch

import crop_goldens
from oracle import crop_transform as ct

TARGETS = [(32, 128), (224, 224)]
ROTATIONS = [0, 90, 180, 270]
# 1 x 1, 1 x N, N x 1, the tall-crop pass order (h > 100 w and the height shrinks: 101 x 1, 268 x 2, 3000 x 3),
# unchanged axes (32 or 128 / 224 on a side), ordinary and large ratios
SWEEP = [(1, 1), (1, 300), (300, 1), (101, 1), (100, 1), (268, 2), (3000, 3), (32, 128), (32, 77), (90, 128),
         (224, 224), (224, 31), (7, 13), (64, 500), (128, 32), (17, 4000)]


def _pil(img, size, rotation):
    Image = pytest.importorskip("PIL.Image")
    T = pytest.importorskip("torchvision.transforms")
    pil = Image.fromarray(img)
    if rotation:
        pil = pil.rotate(rotation, expand=True)
    return np.asarray(T.Resize(size, T.InterpolationMode.BICUBIC)(pil))


@pytest.mark.parametrize("rotation", ROTATIONS)
@pytest.mark.parametrize("size", TARGETS, ids=["32x128", "224x224"])
def test_oracle_equals_pil(size, rotation):
    rng = np.random.default_rng(rotation + size[0])
    sizes = SWEEP + [(int(rng.integers(1, 200)), int(rng.integers(1, 600))) for _ in range(12)]
    for h, w in sizes:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = _pil(img, size, rotation)
        assert np.array_equal(ct.transform_u8(img, size, rotation), ref), (h, w)


def test_oracle_float_output_equals_torchvision():
    Image = pytest.importorskip("PIL.Image")
    T = pytest.importorskip("torchvision.transforms")
    rng = np.random.default_rng(5)
    tf = T.Compose([T.Resize((32, 128), T.InterpolationMode.BICUBIC), T.ToTensor(), T.Normalize(0.5, 0.5)])
    for h, w in [(40, 170), (3, 9), (268, 2)]:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert np.array_equal(ct.transform(img, (32, 128)), tf(Image.fromarray(img)).numpy())


@pytest.mark.parametrize("name", crop_goldens.NAMES)
def test_oracle_equals_goldens(name):
    """Bytes and floats of every crop, both image sizes, every rotation."""
    crops, g = crop_goldens.load(name)
    assert len(g["cases"]) == 8
    for size, rotation in g["cases"]:
        crop_goldens.reference_stack(crops, g, size, rotation)


def test_goldens_cover_the_demo_images_and_tall_crops():
    crops, demo = crop_goldens.load("demo")
    assert len(demo["names"]) == 6 and (871, 1774, 3) in [a.shape for a in crops]
    crops, seeded = crop_goldens.load("seeded")
    assert {(1, 1), (101, 1), (268, 2)} <= {a.shape[:2] for a in crops}
    assert {r for (_, r) in seeded["cases"]} == set(ROTATIONS)


# ---------------------------------------------------------------- Python packing
def test_pack_crops_layout():
    from parseq_b200.system import pack_crops
    a = torch.arange(2 * 3 * 3, dtype=torch.uint8).reshape(2, 3, 3)
    b = torch.full((1, 5, 3), 7, dtype=torch.uint8)
    data, offsets, sizes = pack_crops([a, b])
    assert offsets.tolist() == [0, 18] and sizes.tolist() == [[2, 3], [1, 5]]
    assert offsets.dtype == torch.int64 and sizes.dtype == torch.int32
    assert torch.equal(data[:18], a.reshape(-1)) and torch.equal(data[18:], b.reshape(-1))


def test_pack_crops_takes_rgb_pil_images():
    Image = pytest.importorskip("PIL.Image")
    from parseq_b200.system import pack_crops
    img = np.random.default_rng(0).integers(0, 256, (4, 6, 3), dtype=np.uint8)
    data, offsets, sizes = pack_crops([Image.fromarray(img), torch.from_numpy(img)])
    assert sizes.tolist() == [[4, 6], [4, 6]] and torch.equal(data[:72], data[72:])
    with pytest.raises(ValueError, match="mode RGB"):
        pack_crops([Image.fromarray(img).convert("L")])


@pytest.mark.parametrize("crops, exc", [
    ([], ValueError),
    (torch.zeros((2, 32, 128, 3), dtype=torch.uint8), TypeError),
    ([torch.zeros((4, 4, 3), dtype=torch.float32)], TypeError),
    ([torch.zeros((4, 4, 4), dtype=torch.uint8)], ValueError),
    ([torch.zeros((4, 4), dtype=torch.uint8)], ValueError),
    ([np.zeros((4, 4, 3), dtype=np.uint8)], TypeError),
], ids=["empty", "tensor_not_list", "float_crop", "four_channels", "two_dims", "numpy_array"])
def test_pack_crops_rejects_malformed_lists(crops, exc):
    from parseq_b200.system import pack_crops
    with pytest.raises(exc):
        pack_crops(crops)


def test_pack_crops_rejects_mixed_devices():
    from parseq_b200.system import pack_crops
    a = torch.zeros((2, 2, 3), dtype=torch.uint8)
    b = torch.zeros((2, 2, 3), dtype=torch.uint8, device="meta")
    with pytest.raises(ValueError, match="one device"):
        pack_crops([a, b])


# ---------------------------------------------------------------- C ABI, host-side checks
@pytest.fixture(scope="module")
def lib():
    from parseq_b200.engine import load_library
    try:
        return load_library()
    except (RuntimeError, OSError) as e:
        pytest.skip(str(e))


def _crops(sizes, data_bytes=None, rotation=0, offsets=None):
    from parseq_b200.engine import CropsC
    sz = np.asarray(sizes, dtype=np.int32).reshape(-1, 2)
    n = (3 * sz[:, 0].astype(np.int64) * sz[:, 1])
    off = np.asarray(offsets, dtype=np.int64) if offsets is not None else np.concatenate([[0], np.cumsum(n)[:-1]])
    buf = np.zeros(max(int(n.sum()), 1), dtype=np.uint8)
    c = CropsC(buf.ctypes.data, int(n.sum()) if data_bytes is None else data_bytes, off.ctypes.data, sz.ctypes.data, rotation)
    return c, (buf, sz, off)


@pytest.mark.parametrize("sizes, kw, msg", [
    ([[0, 5]], {}, "sides must be in"),
    ([[5, 8193]], {}, "sides must be in"),
    ([[4, 4], [2, 2]], {"data_bytes": 50}, "exceeds data_bytes"),
    ([[4, 4]], {"offsets": [-1]}, "exceeds data_bytes"),
    ([[4, 4]], {"rotation": 45}, "rotation"),
], ids=["zero_side", "side_over_8192", "past_data_bytes", "negative_offset", "rotation_45"])
def test_crop_entry_points_reject_bad_metadata_without_a_device(lib, sizes, kw, msg):
    """The metadata is checked before the handle: a NULL handle with bad crops reports the crops."""
    from parseq_b200.engine import ForwardArgsC
    c, keep = _crops(sizes, **kw)
    a = ForwardArgsC(len(sizes), -1, 1, 1, None, None)
    out = (C.c_float * 4)()
    for rc in (lib.parseq_resize_crops(None, len(sizes), C.byref(c), out, None),
               lib.parseq_forward_crops(None, C.byref(a), C.byref(c), out, None, None, None),
               lib.parseq_forward_host_crops(None, C.byref(a), C.byref(c), out, None, None, None)):
        assert rc == -1
        assert msg in lib.parseq_last_error().decode()


def test_crop_entry_points_reject_null_handle_and_teacher_forcing(lib):
    from parseq_b200.engine import ForwardArgsC
    c, keep = _crops([[4, 4]])
    out = (C.c_float * 4)()
    assert lib.parseq_resize_crops(None, 1, C.byref(c), out, None) == -1
    assert "null argument" in lib.parseq_last_error().decode()
    a = ForwardArgsC(1, -1, 1, 1, None, None)
    assert lib.parseq_forward_crops(None, C.byref(a), C.byref(c), out, None, None, None) == -1
    assert "null argument" in lib.parseq_last_error().decode()
    assert lib.parseq_forward_crops(None, C.byref(a), None, out, None, None, None) == -1
    forced = (C.c_int32 * 4)()
    a = ForwardArgsC(1, -1, 1, 1, C.cast(forced, C.c_void_p), None)
    assert lib.parseq_forward_host_crops(None, C.byref(a), C.byref(c), out, None, None, None) == -1
    assert "teacher forcing" in lib.parseq_last_error().decode()
