"""Writes tests/golden/crops/*.pt: raw crops of any size and what the reference's own test transform makes of them,
`SceneTextDataModule.get_transform(img_size, rotation=r)` (strhub/data/module.py:69-82: Image.rotate(r, expand=True),
T.Resize(img_size, BICUBIC), ToTensor, Normalize(0.5, 0.5)), loaded from the reference tree with `pytorch_lightning`
and `.dataset` stubbed (nothing else of the data module is used).  Needs the reference tree and PIL:

    python -m oracle.make_golden_crops

Files (torch.save dicts, kept small: the crops are regenerated or decoded, the outputs stored as SHA-256 digests):
  seeded.pt  ragged crops regenerated from SEEDED_SIZES by `seeded_crops()` (a counter-based hash, no RNG stream whose
             output could change between numpy versions): 1 x 1, 1 x N, N x 1, the tall-crop cases 101 x 1 and 268 x 2,
             crops already at a target side, and sizes of the benchmark's distribution (h 16-128, w 32-512).
  demo.pt    the reference's six demo_images as their original files' bytes (JPEG / PNG), decoded to RGB as read.py
             does (`Image.open(...).convert('RGB')`).
Each holds the digest of every crop's RGB bytes ("crops_sha256") and, per (img_size, rotation) for img_size 32 x 128
and 224 x 224 and every rotation, the digests of every crop's transform output: its uint8 image ("u8_sha256",
[H, W, 3] = round(255 * (float * 0.5 + 0.5)), exact because ToTensor + Normalize(0.5, 0.5) map the bytes one to one)
and its float output ("float_sha256", float32 [3, H, W]).
"""
from __future__ import annotations

import glob
import hashlib
import importlib.util
import io
import os
import sys
import types

import numpy as np
import torch

REF_ROOT = os.environ.get("PARSEQ_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "crops")
ROTATIONS = (0, 90, 180, 270)
SMALL, LARGE = (32, 128), (224, 224)


def load_get_transform():
    """SceneTextDataModule.get_transform of the reference's strhub/data/module.py."""
    pl = types.ModuleType("pytorch_lightning")
    pl.LightningDataModule = object
    ds = types.ModuleType("_ref_data.dataset")
    ds.LmdbDataset = ds.build_tree_dataset = None
    pkg = types.ModuleType("_ref_data")
    pkg.__path__ = []
    saved = {k: sys.modules.get(k) for k in ("pytorch_lightning", "_ref_data", "_ref_data.dataset")}
    sys.modules.update({"pytorch_lightning": pl, "_ref_data": pkg, "_ref_data.dataset": ds})
    try:
        spec = importlib.util.spec_from_file_location("_ref_data.module", os.path.join(REF_ROOT, "strhub/data/module.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return mod.SceneTextDataModule.get_transform


SEEDED_SIZES = [(1, 1), (1, 37), (45, 1), (101, 1), (268, 2), (32, 300), (80, 128), (224, 50), (7, 13),
                (57, 389), (121, 44), (16, 512), (128, 33), (93, 201), (40, 460), (66, 97), (110, 310),
                (3, 110), (87, 5), (113, 64), (29, 29)]


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def pixels(h: int, w: int, seed: int) -> np.ndarray:
    """uint8 [h, w, 3] of splitmix64 of the byte index: the same bytes on every machine and numpy version."""
    z = np.arange(h * w * 3, dtype=np.uint64) + np.array([seed], np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    return (z & np.uint64(255)).astype(np.uint8).reshape(h, w, 3)


def seeded_crops():
    return [pixels(h, w, i + 1) for i, (h, w) in enumerate(SEEDED_SIZES)]


def decode(file_bytes: bytes) -> np.ndarray:
    """A demo image's file bytes -> RGB array, as read.py reads it."""
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(file_bytes)).convert("RGB"))


def cases(get_transform, imgs):
    from PIL import Image
    out = {}
    for size in (SMALL, LARGE):
        for r in ROTATIONS:
            tf = get_transform(size, rotation=r)
            xs = [tf(Image.fromarray(a)) for a in imgs]
            out[(size, r)] = {
                "u8_sha256": [digest(torch.round((x * 0.5 + 0.5) * 255).to(torch.uint8).permute(1, 2, 0).numpy()) for x in xs],
                "float_sha256": [digest(x.numpy()) for x in xs]}
    return out


def main():
    get_transform = load_get_transform()
    os.makedirs(OUT, exist_ok=True)
    crops = seeded_crops()
    seeded = {"sizes": SEEDED_SIZES, "crops_sha256": [digest(a) for a in crops], "cases": cases(get_transform, crops)}
    torch.save(seeded, os.path.join(OUT, "seeded.pt"))
    paths = sorted(glob.glob(os.path.join(REF_ROOT, "demo_images", "*")))
    files = [open(p, "rb").read() for p in paths]
    imgs = [decode(f) for f in files]
    demo = {"names": [os.path.basename(p) for p in paths],
            "files": [torch.frombuffer(bytearray(f), dtype=torch.uint8) for f in files],
            "crops_sha256": [digest(a) for a in imgs], "cases": cases(get_transform, imgs)}
    torch.save(demo, os.path.join(OUT, "demo.pt"))
    for f in ("seeded.pt", "demo.pt"):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
