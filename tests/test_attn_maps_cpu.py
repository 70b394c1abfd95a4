"""Cross-attention maps without a GPU: the C ABI's struct layout, the centre / box rule of locate, and the mapping of a
point of the img_size image back to the pixels of a rotated, resized crop."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle.crop_transform import transform_u8
from parseq_b200.engine import ForwardArgsC
from parseq_b200.system import attention_centers_boxes, unrotate_boxes, unrotate_points

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "attention")


def test_attn_maps_is_the_last_field_and_defaults_to_null():
    names = [n for n, _ in ForwardArgsC._fields_]
    assert names[-1] == "attn_maps" and names[:-1] == ["batch", "max_length", "decode_ar", "refine_iters", "forced_ids",
                                                      "forced_refine", "class_mask"]
    assert ForwardArgsC.attn_maps.offset == C.sizeof(ForwardArgsC) - C.sizeof(C.c_void_p)
    a = ForwardArgsC(4, -1, 1, 1, None, None)              # the positional construction of older callers
    assert a.class_mask is None and a.attn_maps is None
    hdr = open(os.path.join(ROOT, "include", "parseq_b200.h")).read()
    body = re.search(r"typedef struct parseq_forward_args \{(.*?)\} parseq_forward_args;", hdr, re.S).group(1)
    fields = re.findall(r"^\s*(?:const\s+)?\w+\*?\s+\**(\w+);", body, re.M)
    assert fields == ["batch", "max_length", "decode_ar", "refine_iters", "forced_ids", "forced_refine", "class_mask",
                      "attn_maps"]


def test_centers_and_boxes_of_hand_made_maps():
    ph, pw = 4, 8
    m = torch.zeros((3, 8, 16))
    m[0, 2, 5] = 1.0                                          # one cell
    m[1, 1, 3], m[1, 1, 4] = 0.75, 0.25                       # two cells of one row
    m[2, 0, 0], m[2, 7, 15], m[2, 3, 3] = 0.5, 0.3, 0.2       # corners and a weak cell
    centers, boxes = attention_centers_boxes(m, (ph, pw), threshold=0.5)
    assert torch.allclose(centers[0], torch.tensor([5.5 * pw, 2.5 * ph]))
    assert boxes[0].tolist() == [5 * pw, 2 * ph, 6 * pw, 3 * ph]
    assert torch.allclose(centers[1], torch.tensor([(0.75 * 3.5 + 0.25 * 4.5) * pw, 1.5 * ph]))
    assert boxes[1].tolist() == [3 * pw, ph, 4 * pw, 2 * ph]          # 0.25 < 0.5 * 0.75: only the strong cell
    cx = (0.5 * 0.5 + 0.3 * 15.5 + 0.2 * 3.5) * pw
    cy = (0.5 * 0.5 + 0.3 * 7.5 + 0.2 * 3.5) * ph
    assert torch.allclose(centers[2], torch.tensor([cx, cy]))
    assert boxes[2].tolist() == [0, 0, 16 * pw, 8 * ph]               # 0.3 >= 0.25 keeps the far corner
    _, loose = attention_centers_boxes(m[2:], (ph, pw), threshold=0.3)
    assert loose[0].tolist() == [0, 0, 16 * pw, 8 * ph]
    _, tight = attention_centers_boxes(m[2:], (ph, pw), threshold=0.9)
    assert tight[0].tolist() == [0, 0, pw, ph]


@pytest.mark.parametrize("rotation", (0, 90, 180, 270))
@pytest.mark.parametrize("hw", ((40, 150), (17, 300), (90, 60)))
def test_points_map_back_through_rotation_and_resize(rotation, hw):
    """A one-pixel marker goes through the reference transform (oracle/crop_transform.py: np.rot90 == PIL's
    Image.rotate(r, expand=True), then PIL's bicubic resize); the centre of the brightest resized pixel, mapped back,
    lands within one resized pixel's footprint of the marker's centre."""
    H, W = 32, 128
    h, w = hw
    rng = np.random.default_rng(rotation + h)
    for _ in range(6):
        y, x = int(rng.integers(2, h - 2)), int(rng.integers(2, w - 2))
        crop = np.zeros((h, w, 3), dtype=np.uint8)
        crop[y, x] = 255
        out = transform_u8(crop, (H, W), rotation)[..., 0].astype(np.int64)
        r, c = np.unravel_index(int(out.argmax()), out.shape)
        back = unrotate_points(torch.tensor([c + 0.5, r + 0.5], dtype=torch.float64), (h, w), (H, W), rotation)
        rh, rw = (w, h) if rotation in (90, 270) else (h, w)
        fx, fy = rw / W, rh / H                                   # a resized pixel in rotated-crop pixels
        if rotation in (90, 270):
            fx, fy = fy, fx
        assert abs(float(back[0]) - (x + 0.5)) <= max(fx, 1.0), (rotation, hw, (x, y), back)
        assert abs(float(back[1]) - (y + 0.5)) <= max(fy, 1.0), (rotation, hw, (x, y), back)


def test_boxes_map_back_to_ordered_corners():
    b = torch.tensor([[8.0, 4.0, 24.0, 12.0]])
    for rot in (0, 90, 180, 270):
        out = unrotate_boxes(b, (40, 150), (32, 128), rot)
        assert bool((out[:, 2:] >= out[:, :2]).all())
        corners = unrotate_points(torch.tensor([[8.0, 4.0], [24.0, 12.0], [8.0, 12.0], [24.0, 4.0]]), (40, 150),
                                  (32, 128), rot)
        assert torch.allclose(out[0, :2], corners.amin(0)) and torch.allclose(out[0, 2:], corners.amax(0))


def test_golden_set_covers_the_issue_cases():
    from make_golden_attention import CASES, GOLDEN_FILE_LIMIT
    names = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.endswith(".pt"))
    assert names == sorted(c[0] for c in CASES)
    blobs = {n: torch.load(os.path.join(GOLDEN, n + ".pt")) for n in names}
    for n in names:
        assert os.path.getsize(os.path.join(GOLDEN, n + ".pt")) < GOLDEN_FILE_LIMIT
    kinds = {(b["experiment"], b["dec_depth"], b["max_label_length"], b["decode_ar"], b["refine_iters"]) for b in
             blobs.values()}
    assert ("parseq", 1, 25, True, 1) in kinds and ("parseq", 1, 25, True, 0) in kinds
    assert ("parseq", 1, 25, False, 0) in kinds and ("parseq", 1, 25, False, 2) in kinds
    assert ("parseq-tiny", 1, 25, True, 1) in kinds and ("parseq", 1, 63, True, 1) in kinds
    assert ("parseq", 2, 25, True, 1) in kinds
    assert any(b["experiment"] == "parseq-patch16-224" and b["maps"].shape[-1] == 196 for b in blobs.values())
    assert any(b["n_extra"] == 2906 and b["allowlist"] is not None for b in blobs.values())
    exits = [b for b in blobs.values() if b["decode_ar"] and not b["refine_iters"] and b["max_length"] is None]
    assert exits and all(b["steps"] < b["max_label_length"] + 1 for b in exits)


@pytest.mark.parametrize("name", sorted(f[:-3] for f in os.listdir(GOLDEN) if f.endswith(".pt")))
def test_golden_maps_are_distributions_and_regenerate(name):
    from make_golden_attention import golden_state_dict
    from make_golden_long import make_config_long
    from parseq_b200.weights import state_dict_digest
    b = torch.load(os.path.join(GOLDEN, name + ".pt"))
    m = b["maps"]
    assert m.dtype == torch.float64 and m.shape == (b["batch"], b["steps"], m.shape[-1])
    assert bool((m >= 0).all())
    assert float((m.sum(-1) - 1).abs().max()) <= 1e-12
    assert b["ids"].shape == (b["batch"], b["steps"])
    img = (224, 224) if b["experiment"] == "parseq-patch16-224" else (32, 128)
    cfg = make_config_long(b["experiment"], b["max_label_length"], b["n_extra"], img_size=img, dec_depth=b["dec_depth"])
    assert m.shape[-1] == cfg.num_patches
    assert state_dict_digest(golden_state_dict(cfg, b["weight_seed"], b["sharp"], b["eos_bias"])) == b["sd_digest"]
