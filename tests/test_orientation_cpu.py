"""Orientation search and per-crop rotations without a GPU: the fp64 rule of tests/orientation_oracle.py, its
confidence against the reference's own `_eval_step` decode, the argument checks of the Python surface, and the host
checks of parseq_forward_crops_oriented / per-crop `rotations` on a NULL handle."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import orientation_oracle as oo


# ---------------------------------------------------------------- the rule
def test_rule_ties_nan_and_threshold():
    assert oo.choose([0.5]) == 0
    assert oo.choose([0.5, 0.5, 0.5, 0.5]) == 0                    # ties keep the earlier orientation
    assert oo.choose([0.2, 0.7, 0.7, 0.1]) == 1
    assert oo.choose([0.2, 0.1, 0.3, 0.9]) == 3
    assert oo.choose([math.nan, 0.0]) == 1                          # NaN ranks below every number
    assert oo.choose([0.0, math.nan, 0.1]) == 2
    assert oo.choose([math.nan, math.nan]) == 0
    assert oo.choose([0.3, 0.9], min_confidence=0.3) == 0          # >= t keeps the first reading
    assert oo.choose([0.3, 0.9], min_confidence=0.31) == 1
    assert oo.choose([math.nan, 0.9], min_confidence=0.0) == 1     # NaN is never >= t
    pick, rr = oo.select(np.array([[0.9, 0.95], [0.1, 0.2], [0.5, 0.4]]), 0.5)
    assert pick.tolist() == [0, 1, 0] and rr.tolist() == [False, True, False]
    pick, rr = oo.select(np.array([[0.9, 0.95], [0.1, 0.2]]))
    assert pick.tolist() == [1, 1] and rr.all()


def _torch_eval_step_confidence(logits: torch.Tensor, decode):
    """base.py:132-142 in fp64: softmax, the tokenizer's decode (ids and probabilities through the EOS), prod."""
    probs = logits.double().softmax(-1)
    _, p = decode(probs)
    return [float(x.prod()) for x in p]


def test_confidence_equals_the_reference_decode():
    """The oracle's confidence is the product the reference's own Tokenizer.decode returns (the EOS probability
    included), for labels that end early, run to the last position, and rows without a finite maximum."""
    from oracle import reference_loader
    if not reference_loader.available():
        pytest.skip("the reference tree is not available")
    _, RefTokenizer = reference_loader.load_reference_classes()
    tok = RefTokenizer("0123456789abcdefghijklmnopqrstuvwxyz")
    C_ = len(tok) - 2
    g = torch.Generator().manual_seed(3)
    x = torch.randn((24, 26, C_), generator=g, dtype=torch.float64) * 3
    x[:8, :, 0] -= 50                                               # no EOS anywhere: the product runs over all rows
    x[8:16, :4, 0] -= 50
    x[8:16, 4, 0] += 50                                             # EOS at position 4
    want = _torch_eval_step_confidence(x, tok.decode)
    got = [oo.reference_confidence(r.numpy())[0] for r in x]
    np.testing.assert_allclose(got, want, rtol=1e-12)
    assert [oo.reference_confidence(r.numpy())[1] for r in x[8:16]] == [4] * 8
    y = x[:2].clone()
    y[0, 0, 3] = math.inf
    y[1, 0, 3] = math.nan
    assert all(math.isnan(oo.reference_confidence(r.numpy())[0]) for r in y)


# ---------------------------------------------------------------- Python surface
@pytest.fixture(scope="module")
def system():
    from parseq_b200.factory import create_model
    return create_model("parseq-tiny")


@pytest.mark.parametrize("orientations", [(), (0, 90, 180, 270, 0), (0, 45), (90, 90), (0, 90, 180, 270, 90), (True,)],
                         ids=["R0", "R5", "45", "duplicate", "R5_dup", "bool"])
def test_bad_orientations(system, orientations):
    crops = [torch.zeros((8, 20, 3), dtype=torch.uint8)]
    with pytest.raises(ValueError, match="orientations must be 1 to 4 distinct values"):
        system.read_oriented(crops, orientations)


def test_tensor_input_and_rotation_arguments(system):
    with pytest.raises(ValueError, match="list of raw crops"):
        system.read_oriented(torch.zeros((2, 3, 32, 128)))
    from parseq_b200.system import _crop_rotations, _reject_tensor_rotation
    assert _crop_rotations(90, 3) == (90, None)
    r, rots = _crop_rotations([0, 90, 270], 3)
    assert rots.dtype == torch.int32 and rots.tolist() == [0, 90, 270]
    with pytest.raises(ValueError, match="one int per crop"):
        _crop_rotations([0, 90], 3)
    for rot in (90, [0, 0], (0,)):
        with pytest.raises(ValueError, match="a tensor input is already at img_size"):
            _reject_tensor_rotation(rot)
    _reject_tensor_rotation(0)
    with pytest.raises(ValueError, match="a tensor input is already at img_size"):
        system.forward(torch.zeros((2, 3, 32, 128)), rotation=[0, 0])
    with pytest.raises(ValueError, match="rotation and orientations cannot be combined"):
        system.locate([torch.zeros((8, 20, 3), dtype=torch.uint8)], rotation=90, orientations=(0, 180))
    with pytest.raises(ValueError, match="min_confidence needs orientations"):
        system.locate([torch.zeros((8, 20, 3), dtype=torch.uint8)], min_confidence=0.5)


def test_max_batch_below_readings_per_crop():
    from parseq_b200.factory import create_model
    m = create_model("parseq-tiny")
    m.model.set_engine_option("max_batch", 2)
    with pytest.raises(ValueError, match=r"max_batch \(2\) must be >= len\(orientations\) - 1 \(3\)"):
        m.read_oriented([torch.zeros((8, 20, 3), dtype=torch.uint8)], (0, 90, 180, 270))


# ---------------------------------------------------------------- C ABI, host-side checks
@pytest.fixture(scope="module")
def lib():
    from parseq_b200.engine import load_library
    try:
        return load_library()
    except (RuntimeError, OSError) as e:
        pytest.skip(str(e))


def _crops(n=2, rotations=None):
    from parseq_b200.engine import CropsC
    sz = np.tile(np.array([[4, 6]], dtype=np.int32), (n, 1))
    off = np.arange(n, dtype=np.int64) * 72
    buf = np.zeros(72 * n, dtype=np.uint8)
    rot = np.asarray(rotations, dtype=np.int32) if rotations is not None else None
    c = CropsC(buf.ctypes.data, buf.size, off.ctypes.data, sz.ctypes.data, 0, rot.ctypes.data if rot is not None else None)
    return c, (buf, sz, off, rot)


def test_per_crop_rotations_are_checked_without_a_device(lib):
    from parseq_b200.engine import ForwardArgsC
    c, keep = _crops(3, [0, 90, 45])
    a = ForwardArgsC(3, -1, 1, 1, None, None)
    out = (C.c_float * 4)()
    for rc in (lib.parseq_resize_crops(None, 3, C.byref(c), out, None),
               lib.parseq_forward_crops(None, C.byref(a), C.byref(c), out, None, None, None),
               lib.parseq_forward_host_crops(None, C.byref(a), C.byref(c), out, None, None, None)):
        assert rc == -1
        assert "crop 2: rotation must be 0, 90, 180 or 270, got 45" in lib.parseq_last_error().decode()
    # a valid list passes the metadata checks and stops at the handle; the uniform field is then ignored
    c, keep = _crops(3, [0, 90, 270])
    c.rotation = 45
    assert lib.parseq_forward_crops(None, C.byref(a), C.byref(c), out, None, None, None) == -1
    assert lib.parseq_last_error().decode() == "null argument"


@pytest.mark.parametrize("orient, msg", [
    (dict(n=0), "num_orientations must be in [1, 4], got 0"),
    (dict(n=5), "num_orientations must be in [1, 4], got 5"),
    (dict(n=2, o=[0, 45]), "orientations must be 0, 90, 180 or 270, got 45"),
    (dict(n=3, o=[0, 180, 0]), "orientations must be distinct, 0 repeats"),
    (dict(n=2, rot_out=False), "null rotation_out or confidence_out"),
    (dict(n=2, rotations=[0, 90]), "rotations must be NULL"),
], ids=["R0", "R5", "45", "duplicate", "null_out", "with_rotations"])
def test_oriented_entry_checks_without_a_device(lib, orient, msg):
    from parseq_b200.engine import ForwardArgsC, orient_args
    c, keep = _crops(2, orient.get("rotations"))
    a = ForwardArgsC(2, -1, 1, 1, None, None)
    out = (C.c_float * 4)()
    rot = (C.c_int32 * 2)()
    conf = (C.c_float * 2)()
    o = orient_args((orient.get("o") or [0, 90, 180, 270, 0])[:max(orient["n"], 0)], None,
                    C.cast(rot, C.c_void_p) if orient.get("rot_out", True) else None, C.cast(conf, C.c_void_p))
    o.num_orientations = orient["n"]
    assert lib.parseq_forward_crops_oriented(None, C.byref(a), C.byref(c), C.byref(o), out, None, None, None) == -1
    assert msg in lib.parseq_last_error().decode()


def test_oriented_entry_reaches_the_handle_check(lib):
    from parseq_b200.engine import ForwardArgsC, orient_args
    c, keep = _crops(2)
    a = ForwardArgsC(2, -1, 1, 1, None, None)
    out = (C.c_float * 4)()
    rot = (C.c_int32 * 2)()
    conf = (C.c_float * 2)()
    o = orient_args((180, 0), 0.5, C.cast(rot, C.c_void_p), C.cast(conf, C.c_void_p))
    assert lib.parseq_forward_crops_oriented(None, C.byref(a), C.byref(c), C.byref(o), out, None, None, None) == -1
    assert lib.parseq_last_error().decode() == "null argument"


def test_scalar_rotations_and_threshold_types(system):
    """A 0-d tensor or numpy scalar is one rotation for every crop, as an int is; min_confidence takes any real scalar
    (numpy, 0-d tensor) but not a bool or a sequence.  Valid arguments get past the checks to the device check."""
    from parseq_b200.system import _crop_rotations, _reject_tensor_rotation
    assert _crop_rotations(torch.tensor(90), 3) == (90, None)
    assert _crop_rotations(np.int64(180), 2) == (180, None)
    assert _crop_rotations(np.array(270), 2) == (270, None)
    _reject_tensor_rotation(torch.tensor(0))
    _reject_tensor_rotation(np.array(0))
    with pytest.raises(ValueError, match="a tensor input is already at img_size"):
        _reject_tensor_rotation(torch.tensor(90))
    crops = [torch.zeros((8, 20, 3), dtype=torch.uint8)]
    for t in (True, [0.5], "0.5", torch.tensor([0.5, 0.2])):
        with pytest.raises(ValueError, match="min_confidence must be None or a real number"):
            system.read_oriented(crops, (0, 180), min_confidence=t)
    for t in (np.float32(0.25), torch.tensor(0.25, dtype=torch.float64), 1, 0.5):
        with pytest.raises(RuntimeError, match="CUDA"):
            system.read_oriented(crops, (0, 180), min_confidence=t)


@pytest.mark.parametrize("case", ["or_s_sharp", "or_ti_c3001", "or_vitstr_s"])
def test_goldens_follow_the_rule(case):
    """tests/golden/orientation: the recorded choice is the fp64 rule applied to the recorded reference confidences,
    each confidence is a product of probabilities, and the goldens are not all upright (the rule is exercised)."""
    import os
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "orientation", case + ".pt"),
                   weights_only=False)
    conf = g["confidence"].T.numpy()
    pick, rr = oo.select(conf)
    assert rr.all() and pick.tolist() == g["chosen"].tolist()
    assert ((conf >= 0) & (conf <= 1)).all()
    assert (g["chosen"] != 0).any()
    R, N, L = g["ids"].shape
    for k in range(R):
        for b in range(N):
            n = int(g["length"][k, b])
            row = g["ids"][k, b]
            if n < g["steps"][k]:
                assert int(row[n]) == 0 and (row[:n] > 0).all()      # the label, then EOS
