"""Loads tests/golden/crops/*.pt (written by oracle/make_golden_crops.py): the crops, regenerated (seeded.pt) or decoded
from the demo images' file bytes (demo.pt) and checked against their recorded digests, and the digests of what the
reference's own transform made of them.  `reference_stack` returns the transform's uint8 / float outputs, recomputed by
the CPU oracle and checked against those digests, so the GPU tests can feed them to the engine."""
import os

import numpy as np
import torch

from oracle import crop_transform as ct
from oracle.make_golden_crops import decode, digest, seeded_crops

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "crops")
NAMES = ("seeded", "demo")


def load(name):
    """(crops: list of uint8 [h, w, 3] arrays, golden dict)."""
    g = torch.load(os.path.join(GOLDEN, f"{name}.pt"), weights_only=False)
    if name == "seeded":
        crops = seeded_crops()
    else:
        crops = [decode(f.numpy().tobytes()) for f in g["files"]]
    got = [digest(a) for a in crops]
    assert got == g["crops_sha256"], f"{name}: the golden crops do not regenerate / decode to the recorded bytes"
    return crops, g


def reference_stack(crops, g, size, rotation):
    """uint8 [N, H, W, 3] and float32 [N, 3, H, W] of the reference transform, as recorded in the golden."""
    case = g["cases"][(tuple(size), rotation)]
    u8 = [ct.transform_u8(a, size, rotation) for a in crops]
    fl = [ct.to_float(x) for x in u8]
    assert [digest(x) for x in u8] == case["u8_sha256"], (size, rotation)
    assert [digest(x) for x in fl] == case["float_sha256"], (size, rotation)
    return torch.from_numpy(np.stack(u8)), torch.from_numpy(np.stack(fl))
