"""Drop-in Python surface of the PARSeq inference path.

`PARSeq` mirrors `strhub.models.parseq.system.PARSeq` (system.py:33-88: ctor kwargs, `.model`,
`.tokenizer`, `.hparams`, `forward(images, max_length)`) and the bits of `BaseSystem` its callers use
(`test_step` -> `BatchResult`, base.py:36-44,112-143,179-180; `.device`).  `ParseqModel` mirrors the
inner `strhub.models.parseq.model.PARSeq` (model.py:31-169): same parameter names (so released
`parseq-*.pt` state_dicts load), `encode`, `forward(tokenizer, images, max_length)`, `decode_ar`,
`refine_iters`, `max_label_length`.  All arithmetic happens in libparseq_b200.so (sm_90a CUDA);
these classes only own the parameters and marshal pointers.  There is no CPU or eager-PyTorch
fallback: calling forward with non-CUDA tensors raises.
"""
from __future__ import annotations

import math
import numbers
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
from torch import Tensor, nn

from .config import ParseqConfig, make_config
from .engine import CropsC, Engine, EngineError
from .lexicon import Lexicon, check_words, lexicon_rows
from .tokenizer import CharsetAdapter, Tokenizer


class InvalidModelError(RuntimeError):
    """Raised for any model-related error (creation, loading) — name kept from strhub/models/utils.py:10."""


@dataclass
class BatchResult:          # base.py:36-44
    num_samples: int
    correct: int
    ned: float
    confidence: float
    label_length: int
    loss: Optional[Tensor]
    loss_numel: Optional[int]


def edit_distance(a: str, b: str) -> int:
    """Levenshtein distance (the reference uses nltk.edit_distance, base.py:29,139)."""
    if a == b:
        return 0
    if not a or not b:
        return len(a) + len(b)
    prev = list(range(len(b) + 1))
    for i, ca in enumerate(a, 1):
        cur = [i]
        for j, cb in enumerate(b, 1):
            cur.append(min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (ca != cb)))
        prev = cur
    return prev[-1]


def _crop_tensor(c) -> Tensor:
    """A raw crop as a uint8 [h, w, 3] tensor: a tensor as given, or the pixels of a PIL image in mode RGB."""
    if isinstance(c, Tensor):
        if c.dtype != torch.uint8:
            raise TypeError(f"a crop must be a uint8 tensor, got {c.dtype}")
        if c.dim() != 3 or c.shape[2] != 3:
            raise ValueError(f"a crop must be [h, w, 3] (HWC RGB), got {tuple(c.shape)}")
        return c
    try:
        from PIL import Image
    except ImportError:             # pragma: no cover
        Image = None
    if Image is not None and isinstance(c, Image.Image):
        if c.mode != "RGB":
            raise ValueError(f"a PIL crop must be in mode RGB, got {c.mode} (convert it, as read.py does)")
        import numpy as np
        return torch.from_numpy(np.asarray(c).copy())
    raise TypeError(f"a crop must be a uint8 [h, w, 3] tensor or a PIL image, got {type(c).__name__}")


class RegionCrops(list):
    """The rectified crops of crop_regions: a list of M CUDA uint8 [h, w, 3] views into one packed buffer, so it goes
    wherever a list of raw crops goes (pack_crops then passes the buffer on without a copy).  Also holds each region's
    `quads` (float64 [M, 4, 2], TL, TR, BR, BL in frame pixels; for a polygon p_0, p_{k-1}, q_0, q_{k-1}), `coeffs`
    (float64 [M, 8], PIL PERSPECTIVE order; NaN for a polygon), `frame_index` (int64 [M]), `polygons` (per region the
    caller's float64 [2k, 2] points of a polygon, else None) and `tps` (per region its TPS coefficients float64
    [2k + 3, 2], else None).  In a call that mixes quads and polygons the quad crops come first in the buffer, so
    `offsets` need not increase."""

    def __init__(self, views: List[Tensor], data: Tensor, offsets: Tensor, sizes: Tensor, quads: Tensor, coeffs: Tensor,
                 frame_index: Tensor, polygons: Optional[List[Optional[Tensor]]] = None,
                 tps: Optional[List[Optional[Tensor]]] = None):
        super().__init__(views)
        self._views = tuple(views)
        self.data, self.offsets, self.sizes = data, offsets, sizes
        self.quads, self.coeffs, self.frame_index = quads, coeffs, frame_index
        self.polygons = list(polygons) if polygons is not None else [None] * len(views)
        self.tps = list(tps) if tps is not None else [None] * len(views)

    def packed(self) -> bool:
        """The list still holds exactly the views of `data` it was made with."""
        return len(self) == len(self._views) and all(a is b for a, b in zip(self, self._views))

    def to_frame(self, points, i: int) -> Tensor:
        """Points (x, y) [..., 2] in the pixels of crop i (pixel j covers [j, j + 1); e.g. locate's centres, or the
        corners of a box) -> the same points in frame pixels, float64, through region i's map (the thin-plate spline
        of a polygon region)."""
        from .regions import map_points, map_tps
        p = points if isinstance(points, Tensor) else torch.as_tensor(points)
        p = p.to(torch.float64)
        if p.shape[-1] != 2:
            raise ValueError(f"points must be [..., 2], got {tuple(p.shape)}")
        i = int(i)
        if self.tps[i] is not None:
            h, w = (int(v) for v in self.sizes[i])
            x, y = map_tps(self.tps[i], h, w, p[..., 0], p[..., 1])
        else:
            x, y = map_points(self.coeffs[i].tolist(), p[..., 0], p[..., 1])
        return torch.stack([x, y], dim=-1)


def pack_crops(crops: Sequence[Any], pin_memory: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    """Packs a list of raw crops of any size for the engine's crop entry points: (data, offsets, sizes), with data the
    crops' HWC bytes back to back on the crops' device (pinned if asked, for CPU crops), offsets int64 [N] and sizes
    int32 [N, 2] = (h, w) on the CPU.  All crops must be on one device; PIL images count as CPU crops.  The crops of
    crop_regions are already packed: their buffer is returned as it is."""
    if isinstance(crops, RegionCrops) and crops.packed():
        return crops.data, crops.offsets, crops.sizes
    if not isinstance(crops, (list, tuple)):
        raise TypeError("crops must be a list of uint8 [h, w, 3] tensors or PIL images")
    if len(crops) == 0:
        raise ValueError("empty crop list")
    ts = [_crop_tensor(c) for c in crops]
    devs = {t.device for t in ts}
    if len(devs) != 1:
        raise ValueError(f"all crops must be on one device, got {sorted(str(d) for d in devs)}")
    sizes = torch.tensor([[t.shape[0], t.shape[1]] for t in ts], dtype=torch.int32)
    nbytes = sizes[:, 0].to(torch.int64) * sizes[:, 1].to(torch.int64) * 3
    offsets = torch.zeros(len(ts), dtype=torch.int64)
    if len(ts) > 1:
        offsets[1:] = torch.cumsum(nbytes, 0)[:-1]
    dev = ts[0].device
    if dev.type == "cuda":
        data = torch.cat([t.reshape(-1) for t in ts])
    else:
        data = torch.empty(int(nbytes.sum()), dtype=torch.uint8, pin_memory=pin_memory)
        for t, o, n in zip(ts, offsets.tolist(), nbytes.tolist()):
            data[o:o + n].copy_(t.reshape(-1))
    return data, offsets, sizes


Allowlist = Union[None, str, Sequence[Optional[str]]]


def allowlist_mask(tokenizer: Tokenizer, allowlist: Allowlist, batch: int, num_classes: int) -> Optional[Tensor]:
    """The engine's per-image class allowlist (parseq_forward_args.class_mask) as CPU int32 [batch, ceil(C / 32)] words:
    bit c % 32 of word c / 32 of row b allows head class c (= token id c) for image b.  `allowlist` is None (no
    constraint: None is returned), one string for every image, or one Optional[str] per image (None: every class).  EOS
    is always allowed, so an empty string decodes to the empty label."""
    if allowlist is None:
        return None
    if isinstance(allowlist, str):
        rows: List[Optional[str]] = [allowlist] * batch
    else:
        rows = list(allowlist)
        if len(rows) != batch:
            raise ValueError(f"allowlist has {len(rows)} entries for {batch} images")
        if all(r is None for r in rows):
            return None
    words = (num_classes + 31) // 32
    bits = torch.zeros((batch, words * 32), dtype=torch.bool)
    cache: Dict[str, Tensor] = {}
    for b, r in enumerate(rows):
        if r is None:
            bits[b, :num_classes] = True
            continue
        if not isinstance(r, str):
            raise TypeError(f"allowlist entry {b} must be a string or None, got {type(r).__name__}")
        if r not in cache:
            unknown = sorted({ch for ch in r if ch not in tokenizer._stoi or tokenizer._stoi[ch] >= num_classes
                              or tokenizer._stoi[ch] == tokenizer.eos_id})
            if unknown:
                raise ValueError(f"allowlist characters not in charset_train: {''.join(unknown)!r}")
            ids = torch.tensor([tokenizer.eos_id] + tokenizer._tok2ids(r), dtype=torch.long)
            row = torch.zeros(words * 32, dtype=torch.bool)
            row[ids] = True
            cache[r] = row
        bits[b] = cache[r]
    weights = torch.tensor([1 << i for i in range(32)], dtype=torch.int64)
    packed = (bits.view(batch, words, 32).to(torch.int64) * weights).sum(-1)
    return torch.where(packed >= 1 << 31, packed - (1 << 32), packed).to(torch.int32)


Candidates = Union[Sequence[str], Sequence[Sequence[str]]]


def pack_candidates(tokenizer: Tokenizer, candidates: Candidates, batch: int, max_label_length: int,
                    num_classes: int) -> Tuple[Tensor, Tensor, Tensor]:
    """The candidate labels of a score call as the engine takes them (parseq_score_args): CPU int32 targets
    [M, max_label_length + 1] = (c_1..c_n, EOS, 0...), lengths [M] and per_image [batch].  `candidates` is one list of
    strings for every image (a lexicon) or one non-empty list per image; candidates are image-major."""
    shared, rows = lexicon_rows(candidates, batch)
    if shared:
        rows = [candidates] * batch
    words = sorted(set(candidates) if shared else {s for r in rows for s in r})
    check_words(tokenizer, words, max_label_length, num_classes)
    # one target row per distinct word, then a gather: a lexicon shared by 512 images costs one row per word
    L = max_label_length + 1
    index = {s: i for i, s in enumerate(words)}
    table = torch.zeros((len(words), L), dtype=torch.int32)
    for s, i in index.items():
        table[i, :len(s) + 1] = torch.tensor(tokenizer._tok2ids(s) + [tokenizer.eos_id], dtype=torch.int32)
    word_len = torch.tensor([len(s) for s in words], dtype=torch.int32)
    if shared:
        pick = torch.tensor([index[s] for s in candidates], dtype=torch.long).repeat(batch)
    else:
        pick = torch.tensor([index[s] for r in rows for s in r], dtype=torch.long)
    per_image = torch.tensor([len(r) for r in rows], dtype=torch.int32)
    return table[pick], word_len[pick], per_image


BEAM_WIDTH_MAX = 16


def check_beam_width(beam_width) -> int:
    """The beam width of a beam_search call: an int in [1, BEAM_WIDTH_MAX] (ValueError otherwise)."""
    if isinstance(beam_width, bool) or not isinstance(beam_width, int) or not 1 <= beam_width <= BEAM_WIDTH_MAX:
        raise ValueError(f"beam_width must be an int in [1, {BEAM_WIDTH_MAX}], got {beam_width!r}")
    return beam_width


def _mask_ptr(mask: Optional[Tensor]):
    return mask.data_ptr() if mask is not None else None


def _ptr(t: Optional[Tensor]):
    return t.data_ptr() if t is not None else None


def _crops_c(data: Tensor, offsets: Tensor, sizes: Tensor, rotation: int, *, rotations: Optional[Tensor] = None) -> CropsC:
    """parseq_crops of packed crops; `rotations`: CPU int32 [N], each crop's own rotation (kept alive by the result)."""
    c = CropsC(data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), int(rotation), _ptr(rotations))
    c._rotations = rotations
    return c


Rotation = Union[int, Sequence[int]]
ORIENTATIONS = (0, 90, 180, 270)


def _is_rotation_list(rotation: Rotation) -> bool:
    """A sequence of per-crop rotations, as opposed to one number (an int, a numpy scalar, a 0-d array or tensor)."""
    if getattr(rotation, "ndim", None) == 0:
        return False
    return isinstance(rotation, (list, tuple, Tensor)) or hasattr(rotation, "__len__")


def _crop_rotations(rotation: Rotation, n: int) -> Tuple[int, Optional[Tensor]]:
    """`rotation=` of a call on raw crops: one int for every crop, or a sequence of n ints, one per crop -> the
    parseq_crops (rotation, rotations) pair (rotations a CPU int32 [n] tensor, or None)."""
    if not _is_rotation_list(rotation):
        return int(rotation), None
    r = [int(x) for x in (rotation.tolist() if isinstance(rotation, Tensor) else rotation)]
    if len(r) != n:
        raise ValueError(f"rotation must be an int or a sequence of one int per crop ({n}), got {len(r)} values")
    return 0, torch.tensor(r, dtype=torch.int32)


def _rotation_of(rotation: Rotation, b: int) -> int:
    """Crop b's rotation of a `rotation=` argument."""
    if not _is_rotation_list(rotation):
        return int(rotation)
    return int(rotation[b])


def _reject_tensor_rotation(rotation: Rotation):
    if _is_rotation_list(rotation) or rotation:
        raise ValueError("rotation applies to lists of raw crops; a tensor input is already at img_size")


def check_orientations(orientations: Sequence[int]) -> Tuple[int, ...]:
    """The orientations of an orientation search: 1 to 4 distinct values of 0, 90, 180, 270 (ValueError otherwise)."""
    o = tuple(orientations)
    if not 1 <= len(o) <= 4 or any(isinstance(x, bool) or x not in ORIENTATIONS for x in o) or len(set(o)) != len(o):
        raise ValueError(f"orientations must be 1 to 4 distinct values of {ORIENTATIONS}, got {orientations!r}")
    return tuple(int(x) for x in o)


_REGION_FORMS = ("regions must be corners [M, 4, 2], polygons [M, 2k, 2] with 3 <= k <= 32, integer boxes [M, 4], or "
                 "a list of M point arrays [n_i, 2], with M >= 1")


def _region_points(regions) -> List[List[Tuple[float, float]]]:
    """`regions` of crop_regions as M lists of Python float points: a quad (TL, TR, BR, BL) or a polygon of 2k points in
    the caller's order.  Forms: corners [M, 4, 2] or polygons [M, 2k, 2] (any real dtype); integer boxes [M, 4] =
    (x0, y0, x1, y1) with x1 > x0 and y1 > y0; a list of per-region point arrays [n_i, 2] of different lengths."""
    import numpy as np
    from .regions import box_quad

    def arr(r):
        return r.detach().cpu().numpy() if isinstance(r, Tensor) else np.asarray(r)

    if isinstance(regions, (list, tuple)) and len(regions) > 1 and len({np.shape(arr(r)) for r in regions}) > 1:
        out = []
        for i, r in enumerate(regions):
            a = arr(r)
            if a.dtype.kind not in "iuf" or a.ndim != 2 or a.shape[1] != 2:
                raise ValueError(f"region {i}: points must be real [n, 2], got {a.dtype} of shape {tuple(a.shape)}")
            if a.shape[0] != 4 and (a.shape[0] % 2 or not 6 <= a.shape[0] <= 64):
                raise ValueError(f"region {i}: {a.shape[0]} points, a region needs 4 corners or an even count of 6 to "
                                 f"64 polygon points")
            out.append([(float(x), float(y)) for x, y in a.astype(np.float64)])
        return out
    r = arr(regions)
    if r.dtype.kind not in "iuf":
        raise ValueError(f"regions must be real corners [M, 4, 2] or integer boxes [M, 4], got dtype {r.dtype}")
    if r.ndim == 3 and r.shape[2] == 2 and r.shape[0] > 0:
        n = r.shape[1]
        if n == 4 or (n % 2 == 0 and 6 <= n <= 64):
            return [[(float(x), float(y)) for x, y in q] for q in r.astype(np.float64)]
        raise ValueError(f"region 0: {n} points; {_REGION_FORMS}, got shape {tuple(r.shape)}")
    if r.ndim == 2 and r.shape[1] == 4 and r.shape[0] > 0:
        if r.dtype.kind == "f":
            raise ValueError("boxes [M, 4] must be integers; give real-valued regions as corners [M, 4, 2]")
        bad = np.nonzero((r[:, 2] <= r[:, 0]) | (r[:, 3] <= r[:, 1]))[0]
        if bad.size:
            raise ValueError(f"box {int(bad[0])}: {r[bad[0]].tolist()} needs x1 > x0 and y1 > y0")
        return [box_quad(b) for b in r.tolist()]
    raise ValueError(f"{_REGION_FORMS}, got shape {tuple(r.shape)}")


def _crop_hw(c) -> Tuple[int, int]:
    """(h, w) of a raw crop as pack_crops takes it."""
    if isinstance(c, Tensor):
        return int(c.shape[0]), int(c.shape[1])
    if hasattr(c, "size") and not callable(c.size):        # PIL: size = (w, h)
        return int(c.size[1]), int(c.size[0])
    t = _crop_tensor(c)
    return int(t.shape[0]), int(t.shape[1])


def attention_centers_boxes(maps: Tensor, patch_size: Sequence[int], threshold: float = 0.5) -> Tuple[Tensor, Tensor]:
    """Where each map row points, in the pixels of the img_size image: maps fp32 [n, gh, gw] (one row per character)
    -> centers [n, 2] = (x, y), the map-weighted centroid of the patch-cell centres, and boxes [n, 4] = (x0, y0, x1, y1),
    the extent of the cells whose weight is >= threshold * the row's maximum.  Cell (r, c) covers x in [c pw, (c+1) pw),
    y in [r ph, (r+1) ph)."""
    ph, pw = int(patch_size[0]), int(patch_size[1])
    n, gh, gw = maps.shape
    m = maps.to(torch.float32)
    ys = (torch.arange(gh, dtype=torch.float32, device=m.device) + 0.5) * ph
    xs = (torch.arange(gw, dtype=torch.float32, device=m.device) + 0.5) * pw
    tot = m.sum(dim=(1, 2)).clamp_min(torch.finfo(torch.float32).tiny)
    cx = (m.sum(dim=1) * xs).sum(-1) / tot
    cy = (m.sum(dim=2) * ys).sum(-1) / tot
    keep = m >= threshold * m.amax(dim=(1, 2), keepdim=True)
    rows, cols = keep.any(dim=2), keep.any(dim=1)                  # [n, gh], [n, gw]
    r_idx = torch.arange(gh, device=m.device).expand(n, gh)
    c_idx = torch.arange(gw, device=m.device).expand(n, gw)
    r0 = torch.where(rows, r_idx, gh).amin(-1)
    r1 = torch.where(rows, r_idx, -1).amax(-1) + 1
    c0 = torch.where(cols, c_idx, gw).amin(-1)
    c1 = torch.where(cols, c_idx, -1).amax(-1) + 1
    boxes = torch.stack([c0 * pw, r0 * ph, c1 * pw, r1 * ph], dim=-1).to(torch.float32)
    return torch.stack([cx, cy], dim=-1), boxes


def unrotate_points(xy: Tensor, crop_hw: Sequence[int], img_size: Sequence[int], rotation: int) -> Tensor:
    """Points (x, y) [..., 2] in the pixels of the img_size image that get_transform made of a crop of size crop_hw
    (strhub/data/module.py:69-82: Image.rotate(rotation, expand=True), counter-clockwise, then T.Resize(img_size))
    -> the same points in the crop's own pixels: the resize scale is undone per axis, then the rotation."""
    h, w = int(crop_hw[0]), int(crop_hw[1])
    H, W = int(img_size[0]), int(img_size[1])
    rh, rw = (w, h) if rotation in (90, 270) else (h, w)          # the rotated crop's size
    xr = xy[..., 0] * (rw / W)
    yr = xy[..., 1] * (rh / H)
    if rotation == 0:
        x, y = xr, yr
    elif rotation == 90:
        x, y = w - yr, xr
    elif rotation == 180:
        x, y = w - xr, h - yr
    elif rotation == 270:
        x, y = yr, h - xr
    else:
        raise ValueError(f"rotation must be 0, 90, 180 or 270, got {rotation}")
    return torch.stack([x, y], dim=-1)


def unrotate_boxes(boxes: Tensor, crop_hw: Sequence[int], img_size: Sequence[int], rotation: int) -> Tensor:
    """Boxes (x0, y0, x1, y1) [n, 4] of the img_size image -> the crop's pixels (unrotate_points of two corners)."""
    a = unrotate_points(boxes[:, :2], crop_hw, img_size, rotation)
    b = unrotate_points(boxes[:, 2:], crop_hw, img_size, rotation)
    return torch.cat([torch.minimum(a, b), torch.maximum(a, b)], dim=-1)


def _weights_changed(module: nn.Module, *_):
    """Makes the _EngineModule that owns `module` (module.__dict__["_owner"], a weak reference) walk its parameters
    again and upload them on its next engine call.  Runs when a parameter is registered or replaced (which also covers
    load_state_dict(assign=True)) and after every load_state_dict (a load_state_dict post hook): an in-place reload of
    inference tensors changes no version counter and no parameter identity, so the signature alone cannot see it."""
    ref = module.__dict__.get("_owner")
    owner = ref() if ref is not None else None
    if owner is not None:
        owner.__dict__.pop("_plist", None)
        owner.__dict__["_engine_sig"] = None


class _Holder(nn.Module):
    """Parameter container; nested so that state_dict keys equal the reference's."""

    def register_parameter(self, name: str, param: Optional[nn.Parameter]) -> None:
        super().register_parameter(name, param)
        _weights_changed(self)


class _HeadModule(_Holder):
    """`model.head` (model.py:63, nn.Linear(embed_dim, num_tokens - 2)) as a callable: x [..., D] fp32 -> logits."""

    def forward(self, x: Tensor) -> Tensor:
        owner = self.__dict__["_owner"]()
        eng = owner.engine()
        D = owner.cfg.embed_dim
        if x.device.type != "cuda":
            raise RuntimeError("head() takes CUDA tensors (no CPU fallback)")
        x2 = x.to(torch.float32).reshape(-1, D).contiguous()
        out = torch.empty((x2.shape[0], owner.cfg.num_classes), dtype=torch.float32, device=x.device)
        eng.head(x2.shape[0], x2.data_ptr(), out.data_ptr(), torch.cuda.current_stream(x.device).cuda_stream)
        return out.reshape(*x.shape[:-1], owner.cfg.num_classes)


class _TextEmbedModule(_Holder):
    """`model.text_embed` (modules.py:168-176, TokenEmbedding) as a callable: ids [...] -> sqrt(D) * embedding[ids]."""

    def forward(self, tokens: Tensor) -> Tensor:
        owner = self.__dict__["_owner"]()
        eng = owner.engine()
        if tokens.device.type != "cuda":
            raise RuntimeError("text_embed() takes CUDA tensors (no CPU fallback)")
        ids = tokens.to(torch.int32).contiguous()
        out = torch.empty((*ids.shape, owner.cfg.embed_dim), dtype=torch.float32, device=ids.device)
        eng.text_embed(ids.numel(), ids.data_ptr(), out.data_ptr(), torch.cuda.current_stream(ids.device).cuda_stream)
        return out


def _register(root: nn.Module, key: str, tensor: Tensor):
    parts = key.split(".")
    mod = root
    for p in parts[:-1]:
        if not hasattr(mod, p):
            mod.add_module(p, _Holder())
        mod = getattr(mod, p)
    mod.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


class _EngineModule(nn.Module):
    """Owns the parameters (reference state_dict names) and the lazily created engine handle."""

    def __init__(self, cfg: ParseqConfig):
        super().__init__()
        from .weights import init_state_dict
        self.cfg = cfg
        self.max_label_length = cfg.max_label_length
        # random init with the reference's distributions (weights.py); bf16-exact not forced here
        for k, v in init_state_dict(cfg, seed=0, perturb=False, bf16_exact=False).items():
            _register(self, k, v)
        self._engine: Optional[Engine] = None
        self._engine_sig = None
        self._options = {}
        # `head` / `text_embed` are callable like the reference's submodules (they hold the same parameters)
        import weakref
        for name, cls in (("head", _HeadModule), ("text_embed", _TextEmbedModule)):
            if hasattr(self, name):
                getattr(self, name).__class__ = cls
        # every module of the tree reports parameter replacements and reloads to this one (_weights_changed)
        for mod in self.modules():
            mod.__dict__["_owner"] = weakref.ref(self)
            mod.register_load_state_dict_post_hook(_weights_changed)

    # ---- engine plumbing -------------------------------------------------------------------
    @property
    def _device(self) -> torch.device:
        return next(self.parameters()).device

    def register_parameter(self, name: str, param: Optional[nn.Parameter]) -> None:
        super().register_parameter(name, param)
        _weights_changed(self)

    def _signature(self):
        """Cheap staleness check of the engine's weight copy: version counters of every parameter (in-place updates)
        + the storage addresses of the first / last one (`.to()` moves).  The parameter list is cached: walking the
        module tree costs more than a bs=1 forward's launch overhead.  Replaced parameters and load_state_dict reach
        the engine through _weights_changed, which drops the cached list and the signature."""
        pl = self.__dict__.get("_plist")
        if pl is None:
            pl = list(self.parameters())
            self.__dict__["_plist"] = pl
        try:
            vers = tuple(p._version for p in pl)
        except RuntimeError:           # inference tensors carry no version counter
            vers = tuple(id(p) for p in pl)
        return (vers, pl[0].data_ptr(), pl[-1].data_ptr(), len(pl))

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self.__dict__.pop("_plist", None)
        self._engine_sig = None
        return out

    def engine(self) -> Engine:
        """The engine handle, with the current weights uploaded.  The next call after any of these computes with the
        new weights: load_state_dict in any form (strict or not, assign=True, inside or outside inference mode, on
        inference-tensor parameters), replacing a parameter, an in-place update of ordinary parameters (an optimizer
        step), and `.to()`.  Otherwise nothing is uploaded.  One change cannot be seen without reading the weights: an
        in-place write into a parameter that is an inference tensor (built or loaded under torch.inference_mode),
        made outside load_state_dict.  After such a write, call load_state_dict again."""
        dev = self._device
        if dev.type != "cuda":
            raise RuntimeError("parseq_b200 runs on a CUDA (sm_90a, H100) device only; move the model with .to('cuda') "
                               "— there is no CPU fallback")
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        if self._engine is None or self._engine.device != idx:
            self._engine = Engine(self.cfg, idx)
            for name, value in self._options.items():
                self._engine.set_option(name, value)
            self._engine_sig = None
        sig = self._signature()
        if sig != self._engine_sig:
            self._engine.load_state_dict(self.state_dict(), torch.cuda.current_stream(idx).cuda_stream)
            self._engine_sig = sig
        return self._engine

    def set_engine_option(self, name: str, value: int):
        """Engine tuning knobs: "max_batch", "chunk", "use_graph" (see include/parseq_b200.h)."""
        if self._engine is not None:
            self._engine.set_option(name, value)
        self._options[name] = int(value)          # a refused option is not replayed on a later handle

    def _check_images(self, images: Tensor) -> Tensor:
        if images.device.type != "cuda":
            raise RuntimeError("images must be CUDA tensors (no CPU fallback)")
        H, W = self.cfg.img_size
        if images.dtype == torch.uint8:      # raw crops [N, H, W, 3]: ToTensor + Normalize(0.5, 0.5) run inside the engine
            if images.dim() != 4 or tuple(images.shape[1:]) != (H, W, 3):
                raise AssertionError(f"uint8 input must be (N,{H},{W},3), got {tuple(images.shape)}")
            return images.contiguous()
        if images.dim() != 4 or images.shape[1] != 3 or tuple(images.shape[-2:]) != (H, W):
            raise AssertionError(f"Input image size {tuple(images.shape)} doesn't match model (N,3,{H},{W})")
        return images.to(torch.float32).contiguous()

    def _features(self, img: Tensor) -> Tensor:
        """timm forward_features of the ViT: fp32 [N, tokens, D]."""
        eng = self.engine()
        img = self._check_images(img)
        if img.dtype == torch.uint8:
            raise AssertionError("encode / forward_features take normalised float images")
        mem = torch.empty((img.shape[0], self.cfg.enc_tokens, self.cfg.embed_dim), dtype=torch.float32,
                          device=img.device)
        eng.encode(img.data_ptr(), img.shape[0], mem.data_ptr(), torch.cuda.current_stream(img.device).cuda_stream)
        return mem

    def preprocess(self, crops: Sequence[Any], rotation: Rotation = 0) -> Tensor:
        """CUDA uint8 [N, H, W, 3]: each crop rotated by `rotation` (counter-clockwise; one int for every crop or one
        per crop) and resized to img_size on the device, byte-identical to the reference's Image.rotate(rotation,
        expand=True) + T.Resize(img_size, BICUBIC)."""
        eng = self.engine()
        dev = self._device
        data, offsets, sizes = pack_crops(crops, pin_memory=True)
        if data.device.type == "cuda" and data.device != dev:
            raise ValueError(f"crops are on {data.device}, the model on {dev}")
        data = data.to(dev, non_blocking=True)
        H, W = self.cfg.img_size
        out = torch.empty((len(crops), H, W, 3), dtype=torch.uint8, device=dev)
        rot, rots = _crop_rotations(rotation, len(crops))
        eng.resize_crops(_crops_c(data, offsets, sizes, rot, rotations=rots), len(crops), out.data_ptr(),
                         torch.cuda.current_stream(dev).cuda_stream)
        return out

    def crop_regions(self, frames, regions, frame_index=None) -> RegionCrops:
        """Text regions of full frames, rectified on the device (parseq_warp_regions for quads and boxes,
        parseq_warp_polygons for polygons): see _System.crop_regions."""
        from .engine import PolygonsC, RegionsC, tps_coeffs
        from .regions import check_polygon, check_quad, engine_points, polygon_size, quad_coeffs, quad_size
        import numpy as np
        frame_list = list(frames) if isinstance(frames, (list, tuple)) else [frames]
        if not frame_list:
            raise ValueError("no frames")
        regs = _region_points(regions)
        M, F = len(regs), len(frame_list)
        if frame_index is None:
            if F > 1:
                raise ValueError(f"frame_index is required with more than one frame ({F})")
            fidx = np.zeros(M, dtype=np.int64)
        else:
            fi = frame_index.cpu().numpy() if isinstance(frame_index, Tensor) else np.asarray(frame_index)
            if fi.shape != (M,) or fi.dtype.kind not in "iu":
                raise ValueError(f"frame_index must be integer [{M}], got {fi.dtype} {tuple(fi.shape)}")
            if M and (fi.min() < 0 or fi.max() >= F):
                raise ValueError(f"frame_index must be in [0, {F}), got values in [{fi.min()}, {fi.max()}]")
            fidx = fi.astype(np.int64)
        sizes, coeffs, quads, epts = [], [], [], []
        for i, q in enumerate(regs):
            if len(q) == 4:
                check_quad(q, i)
                h, w = quad_size(q)
                coeffs.append(quad_coeffs(q, h, w))
                quads.append(q)
                epts.append(None)
            else:
                check_polygon(q, i)
                e = engine_points(q)
                h, w = polygon_size(e)
                k = len(q) // 2
                coeffs.append((math.nan,) * 8)
                quads.append([q[0], q[k - 1], q[k], q[-1]])
                epts.append(e)
            sizes.append((h, w))
        for f, fr in enumerate(frame_list):
            if isinstance(fr, Tensor) and (fr.dtype != torch.uint8 or fr.dim() != 3 or fr.shape[2] != 3):
                raise ValueError(f"frame {f} must be uint8 [H, W, 3] (HWC RGB), got {fr.dtype} {tuple(fr.shape)}")
            if not isinstance(fr, Tensor) and getattr(fr, "mode", "RGB") != "RGB":
                raise ValueError(f"frame {f}: a PIL frame must be in mode RGB, got {fr.mode}")
        eng = self.engine()
        dev = self._device
        one = frame_list[0]
        if F == 1 and isinstance(one, Tensor) and one.is_cuda:
            fdata = one.contiguous().view(-1)
            foffsets = torch.zeros(1, dtype=torch.int64)
            fsizes = torch.tensor([[one.shape[0], one.shape[1]]], dtype=torch.int32)
        else:
            fdata, foffsets, fsizes = pack_crops(frame_list, pin_memory=True)
        if fdata.device.type == "cuda" and fdata.device != dev:
            raise ValueError(f"frames are on {fdata.device}, the model on {dev}")
        fdata = fdata.to(dev, non_blocking=True)
        # quad crops first, then polygon crops, each group in region order
        qi = [i for i in range(M) if epts[i] is None]
        pi = [i for i in range(M) if epts[i] is not None]
        sz = torch.tensor(sizes, dtype=torch.int32).reshape(M, 2)
        nbytes = 3 * sz[:, 0].to(torch.int64) * sz[:, 1].to(torch.int64)
        order = torch.tensor(qi + pi, dtype=torch.int64)
        offsets = torch.zeros(M, dtype=torch.int64)
        if M > 1:
            offsets[order[1:]] = torch.cumsum(nbytes[order], 0)[:-1]
        total = int(nbytes.sum())
        qbytes = int(nbytes[qi].sum()) if qi else 0
        out = torch.empty(total, dtype=torch.uint8, device=dev)
        cf = torch.tensor(coeffs, dtype=torch.float64).reshape(M, 8)
        stream = torch.cuda.current_stream(dev).cuda_stream
        if qi:
            q_sz = sz[qi].contiguous()
            q_cf = cf[qi].contiguous()
            q_fi = torch.from_numpy(fidx[qi].astype(np.int32))
            rc = RegionsC(fdata.data_ptr(), fdata.numel(), foffsets.data_ptr(), fsizes.data_ptr(), F, q_fi.data_ptr(),
                          q_sz.data_ptr(), q_cf.data_ptr())
            eng.warp_regions(rc, len(qi), out.data_ptr(), qbytes, stream)
        tps = [None] * M
        polys = [None] * M
        if pi:
            p_sz = sz[pi].contiguous()
            p_fi = torch.from_numpy(fidx[pi].astype(np.int32))
            p_np = torch.tensor([len(epts[i]) for i in pi], dtype=torch.int32)
            p_pts = torch.tensor([xy for i in pi for xy in epts[i]], dtype=torch.float64)
            pc = PolygonsC(fdata.data_ptr(), fdata.numel(), foffsets.data_ptr(), fsizes.data_ptr(), F, p_fi.data_ptr(),
                           p_sz.data_ptr(), p_np.data_ptr(), p_pts.data_ptr())
            eng.warp_polygons(pc, len(pi), out.data_ptr() + qbytes, total - qbytes, stream)
            for i in pi:
                polys[i] = torch.tensor(regs[i], dtype=torch.float64)
                tps[i] = torch.from_numpy(tps_coeffs(epts[i], eng.lib))
        views = [out[o:o + 3 * h * w].view(h, w, 3) for o, (h, w) in zip(offsets.tolist(), sizes)]
        return RegionCrops(views, out, offsets, sz, torch.tensor(quads, dtype=torch.float64).reshape(M, 4, 2), cf,
                           torch.from_numpy(fidx), polys, tps)

    def score(self, images: Union[Tensor, List[Any]], targets: Tensor, lengths: Tensor, per_image: Tensor, *,
              rotation: Rotation = 0, return_token_logprobs: bool = False, return_attention: bool = False):
        """Log-likelihoods of candidate labels (parseq_score): `targets` int32 [M, max_label_length + 1] (c_1..c_n, EOS),
        `lengths` [M], `per_image` [N] as pack_candidates makes them (CPU).  Returns fp32 scores [M] on the device, and
        with return_token_logprobs the per-position terms [M, max_label_length + 1] (0 past each label's EOS), with
        return_attention the cross-attention maps fp32 [M, max_label_length + 1, T] (parseq_score_args.attn_maps: row i
        the map of the query predicting t_i, 0 past each label's EOS), in that order.
        `images` as forward takes them; raw crops are resized on the device first (preprocess)."""
        eng = self.engine()
        if isinstance(images, (list, tuple)):
            images = self.preprocess(images, rotation)
        else:
            _reject_tensor_rotation(rotation)
        images = self._check_images(images)
        dev = images.device
        L = self.cfg.max_label_length + 1
        targets = targets.to(device="cpu", dtype=torch.int32).contiguous()
        lengths = lengths.to(device="cpu", dtype=torch.int32).contiguous()
        per_image = per_image.to(device="cpu", dtype=torch.int32).contiguous()
        if targets.dim() != 2 or targets.shape[1] != L or lengths.shape != (targets.shape[0],):
            raise ValueError(f"targets must be int32 [M, {L}] and lengths [M]")
        if per_image.shape != (images.shape[0],):
            raise ValueError(f"per_image must have one entry per image ({images.shape[0]})")
        M = targets.shape[0]
        scores = torch.empty((M,), dtype=torch.float32, device=dev)
        tlp = torch.empty((M, L), dtype=torch.float32, device=dev) if return_token_logprobs else None
        maps = torch.empty((M, L, self.cfg.enc_tokens), dtype=torch.float32, device=dev) if return_attention else None
        eng.score(images.data_ptr(), images.shape[0], per_image, targets, lengths, scores.data_ptr(),
                  tlp.data_ptr() if tlp is not None else None, torch.cuda.current_stream(dev).cuda_stream,
                  u8=images.dtype == torch.uint8, attn_maps_ptr=_ptr(maps))
        out = (scores,) + ((tlp,) if return_token_logprobs else ()) + ((maps,) if return_attention else ())
        return out if len(out) > 1 else scores

    def beam_search(self, images: Union[Tensor, List[Any]], beam_width: int = 5, max_length: Optional[int] = None, *,
                    rotation: Rotation = 0, class_mask: Optional[Tensor] = None, lexicon: Optional[Lexicon] = None,
                    roots: Optional[Tensor] = None, return_attention: bool = False):
        """Beam search (parseq_beam_search): the `beam_width` most likely readings of each image, best first, as raw
        (ids int32 [N, K, num_steps] = c_1..c_n then 0, lengths int32 [N, K] (-1: no hypothesis), scores fp32 [N, K]
        (-inf: no hypothesis)) on the device.  A hypothesis's score is its AR log-likelihood, the quantity `score`
        computes.  `images` as forward takes them; `class_mask`: per-image allowlist words (allowlist_mask).
        `lexicon` (a compiled Lexicon) restricts every hypothesis to its words (parseq_beam_search_lexicon); `roots`:
        CPU int32 [N], the node each image starts at (Lexicon.roots_for), or None for node 0.  return_attention: also
        the hypotheses' cross-attention maps fp32 [N, K, num_steps, T] (parseq_beam_args.attn_maps: `score`'s maps of
        each hypothesis's label, 0 past its EOS and for a missing hypothesis)."""
        check_beam_width(beam_width)
        if lexicon is None and roots is not None:
            raise ValueError("roots need a lexicon")
        if max_length is not None and int(max_length) < 0:
            raise ValueError(f"max_length must be None or >= 0, got {max_length}")
        if lexicon is not None:
            # the trie holds class ids of one charset (which fixes the class count), its words at most one
            # max_label_length long
            if lexicon.charset != self.cfg.charset_train:
                raise ValueError(f"lexicon was compiled for another charset_train ({lexicon.num_classes} classes) than "
                                 f"the model's ({self.cfg.num_classes} classes)")
            if lexicon.max_label_length != self.cfg.max_label_length:
                raise ValueError(f"lexicon was compiled for max_label_length = {lexicon.max_label_length}, the model "
                                 f"has {self.cfg.max_label_length}")
        eng = self.engine()
        if isinstance(images, (list, tuple)):
            images = self.preprocess(images, rotation)
        else:
            _reject_tensor_rotation(rotation)
        images = self._check_images(images)
        dev = images.device
        N, K, S = images.shape[0], int(beam_width), eng.num_steps(max_length)
        if class_mask is not None:
            if tuple(class_mask.shape) != (N, (self.cfg.num_classes + 31) // 32) or class_mask.dtype != torch.int32:
                raise ValueError(f"class_mask must be int32 [{N}, {(self.cfg.num_classes + 31) // 32}]")
            class_mask = class_mask.to(dev, non_blocking=True).contiguous()
        ids = torch.empty((N, K, S), dtype=torch.int32, device=dev)
        lengths = torch.empty((N, K), dtype=torch.int32, device=dev)
        scores = torch.empty((N, K), dtype=torch.float32, device=dev)
        maps = torch.empty((N, K, S, self.cfg.enc_tokens), dtype=torch.float32, device=dev) if return_attention else None
        lex = None
        if lexicon is not None:
            lex = lexicon.handle(eng)
            if roots is not None:
                roots = roots.to(device="cpu", dtype=torch.int32).contiguous()
                if roots.shape != (N,):
                    raise ValueError(f"roots must be int32 [{N}]")
        eng.beam_search(images.data_ptr(), N, K, ids.data_ptr(), lengths.data_ptr(), scores.data_ptr(),
                        torch.cuda.current_stream(dev).cuda_stream, max_length, _mask_ptr(class_mask),
                        u8=images.dtype == torch.uint8, lexicon=lex, roots=roots, attn_maps_ptr=_ptr(maps))
        return (ids, lengths, scores, maps) if return_attention else (ids, lengths, scores)

    def _run_crops(self, crops, max_length, decode_ar, refine_iters, rotation, class_mask=None, attn_maps=False):
        """Raw crops of any size: CUDA crops run parseq_forward_crops and return CUDA tensors; CPU crops and PIL images
        run parseq_forward_host_crops (pinned upload, host outputs) and return CPU tensors.  `class_mask`: the CPU
        allowlist words of allowlist_mask, or None.  attn_maps: also return the fp32 [N, num_steps, T] cross-attention
        maps (else None)."""
        eng = self.engine()
        dev = self._device
        data, offsets, sizes = pack_crops(crops, pin_memory=True)
        host = data.device.type != "cuda"
        if not host and data.device != dev:
            raise ValueError(f"crops are on {data.device}, the model on {dev}")
        N = len(crops)
        L = eng.num_steps(max_length)
        out_dev = torch.device("cpu") if host else dev
        logits = torch.empty((N, L, self.cfg.num_classes), dtype=torch.float32, device=out_dev, pin_memory=host)
        ids = torch.empty((N, L), dtype=torch.int32, device=out_dev, pin_memory=host)
        steps = torch.empty((1,), dtype=torch.int32, device=out_dev, pin_memory=host)
        maps = (torch.empty((N, L, self.cfg.enc_tokens), dtype=torch.float32, device=out_dev, pin_memory=host)
                if attn_maps else None)
        if class_mask is not None:
            class_mask = class_mask.pin_memory() if host else class_mask.to(dev, non_blocking=True)
        rot, rots = _crop_rotations(rotation, N)
        eng.forward_crops(_crops_c(data, offsets, sizes, rot, rotations=rots), N, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(),
                          torch.cuda.current_stream(dev).cuda_stream, max_length, decode_ar, refine_iters, host=host,
                          class_mask_ptr=_mask_ptr(class_mask), attn_maps_ptr=_ptr(maps))
        return logits, ids, steps, maps

    def _run(self, images: Union[Tensor, List[Any]], max_length, decode_ar, refine_iters, forced_ids=None,
             forced_refine=None, rotation: Rotation = 0, class_mask: Optional[Tensor] = None, attn_maps: bool = False):
        """(logits, ids, steps, maps) of one engine forward; maps is None unless attn_maps."""
        if class_mask is not None and (forced_ids is not None or forced_refine is not None):
            raise ValueError("an allowlist cannot be combined with teacher forcing")
        if attn_maps and (forced_ids is not None or forced_refine is not None):
            raise ValueError("attention maps cannot be combined with teacher forcing")
        if isinstance(images, (list, tuple)):
            if forced_ids is not None or forced_refine is not None:
                raise ValueError("teacher forcing takes normalised float images")
            return self._run_crops(images, max_length, decode_ar, refine_iters, rotation, class_mask, attn_maps)
        _reject_tensor_rotation(rotation)
        eng = self.engine()
        images = self._check_images(images)
        dev = images.device
        N = images.shape[0]
        L = eng.num_steps(max_length)
        logits = torch.empty((N, L, self.cfg.num_classes), dtype=torch.float32, device=dev)
        ids = torch.empty((N, L), dtype=torch.int32, device=dev)
        steps = torch.empty((1,), dtype=torch.int32, device=dev)
        maps = torch.empty((N, L, self.cfg.enc_tokens), dtype=torch.float32, device=dev) if attn_maps else None
        fi = forced_ids.to(device=dev, dtype=torch.int32).contiguous() if forced_ids is not None else None
        fr = forced_refine.to(device=dev, dtype=torch.int32).contiguous() if forced_refine is not None else None
        st = torch.cuda.current_stream(dev).cuda_stream
        if class_mask is not None:
            if tuple(class_mask.shape) != (N, (self.cfg.num_classes + 31) // 32) or class_mask.dtype != torch.int32:
                raise ValueError(f"class_mask must be int32 [{N}, {(self.cfg.num_classes + 31) // 32}]")
            class_mask = class_mask.to(dev, non_blocking=True).contiguous()
        if images.dtype == torch.uint8:
            eng.forward_u8(images.data_ptr(), N, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, max_length,
                           decode_ar, refine_iters, class_mask_ptr=_mask_ptr(class_mask), attn_maps_ptr=_ptr(maps))
        else:
            eng.forward(images.data_ptr(), N, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, max_length,
                        decode_ar, refine_iters, fi.data_ptr() if fi is not None else None,
                        fr.data_ptr() if fr is not None else None, _mask_ptr(class_mask), _ptr(maps))
        return logits, ids, steps, maps

    def _run_oriented(self, crops, orientations, min_confidence, max_length, decode_ar, refine_iters, class_mask=None,
                      attn_maps=False):
        """Orientation search over raw crops (parseq_forward_crops_oriented): (logits, ids, steps, maps, rotation int32,
        confidence fp32), on the device for CUDA crops and on the CPU for CPU crops; maps None unless attn_maps."""
        if not isinstance(crops, (list, tuple)):
            raise ValueError("orientation search takes a list of raw crops; a tensor input is already at img_size")
        orientations = check_orientations(orientations)
        if min_confidence is not None:
            scalar = isinstance(min_confidence, numbers.Real) or getattr(min_confidence, "ndim", None) == 0
            if isinstance(min_confidence, bool) or not scalar or getattr(min_confidence, "dtype", None) == torch.bool:
                raise ValueError(f"min_confidence must be None or a real number, got {min_confidence!r}")
            min_confidence = float(min_confidence)
        mb = self._options.get("max_batch")
        if mb is not None and 0 < mb < len(orientations) - 1:
            raise ValueError(f"max_batch ({mb}) must be >= len(orientations) - 1 ({len(orientations) - 1}): a crop's "
                             "readings share one super-chunk")
        eng = self.engine()
        dev = self._device
        data, offsets, sizes = pack_crops(crops, pin_memory=True)
        host = data.device.type != "cuda"
        if not host and data.device != dev:
            raise ValueError(f"crops are on {data.device}, the model on {dev}")
        N = len(crops)
        L = eng.num_steps(max_length)
        logits = torch.empty((N, L, self.cfg.num_classes), dtype=torch.float32, device=dev)
        ids = torch.empty((N, L), dtype=torch.int32, device=dev)
        steps = torch.empty((1,), dtype=torch.int32, device=dev)
        rotation = torch.empty((N,), dtype=torch.int32, device=dev)
        confidence = torch.empty((N,), dtype=torch.float32, device=dev)
        maps = torch.empty((N, L, self.cfg.enc_tokens), dtype=torch.float32, device=dev) if attn_maps else None
        if class_mask is not None:
            class_mask = class_mask.to(dev, non_blocking=True).contiguous()
        eng.forward_crops_oriented(_crops_c(data, offsets, sizes, orientations[0]), N, orientations, min_confidence,
                                   logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), rotation.data_ptr(),
                                   confidence.data_ptr(), torch.cuda.current_stream(dev).cuda_stream, max_length,
                                   decode_ar, refine_iters, class_mask_ptr=_mask_ptr(class_mask), attn_maps_ptr=_ptr(maps))
        out = (logits, ids, steps, maps, rotation, confidence)
        if host:                       # the copies also wait for the call, which reads the pinned crop bytes
            out = tuple(t.cpu() if t is not None else None for t in out)
        return out


class ParseqModel(_EngineModule):
    def __init__(self, cfg: ParseqConfig):
        super().__init__(cfg)
        self.decode_ar = cfg.decode_ar
        self.refine_iters = cfg.refine_iters

    # ---- reference API ---------------------------------------------------------------------
    def encode(self, img: Tensor) -> Tensor:
        return self._features(img)

    @staticmethod
    def _bool_mask(mask: Optional[Tensor], shape, dev) -> Optional[Tensor]:
        """torch's attention masks are bool (True = masked) or additive floats (-inf = masked, 0 = keep)."""
        if mask is None:
            return None
        if mask.dtype == torch.bool:
            m = mask
        elif mask.is_floating_point():
            if bool(((mask != 0) & ~torch.isneginf(mask)).any()):
                raise NotImplementedError("additive attention masks other than 0 / -inf are not supported by the engine")
            m = torch.isneginf(mask)
        else:
            m = mask != 0
        if tuple(m.shape) != tuple(shape):
            raise AssertionError(f"mask shape {tuple(m.shape)} != {tuple(shape)}")
        return m.to(device=dev, dtype=torch.uint8).contiguous()

    def decode(self, tgt: Tensor, memory: Tensor, tgt_mask: Optional[Tensor] = None,
               tgt_padding_mask: Optional[Tensor] = None, tgt_query: Optional[Tensor] = None,
               tgt_query_mask: Optional[Tensor] = None) -> Tensor:
        """model.py:86-103: decoder output [N, NQ, D] (before `head`) for context ids `tgt` [N, J] and encoder `memory`
        [N, T, D].  `tgt_mask` [J, J] acts on the content stream only, which the decoder updates in every layer but
        the last (modules.py:117-123): it is honoured at dec_depth >= 2, and accepted and ignored at depth 1."""
        eng = self.engine()
        dev = memory.device
        if dev.type != "cuda" or tgt.device != dev:
            raise RuntimeError("decode() takes CUDA tensors (no CPU fallback)")
        N, J = tgt.shape
        D, T = self.cfg.embed_dim, self.cfg.enc_tokens
        if tuple(memory.shape) != (N, T, D):
            raise AssertionError(f"memory shape {tuple(memory.shape)} != {(N, T, D)}")
        ids = tgt.to(torch.int32).contiguous()
        mem = memory.to(torch.float32).contiguous()
        q = None
        NQ = J
        if tgt_query is not None:
            NQ = tgt_query.shape[1]
            q = tgt_query.to(device=dev, dtype=torch.float32).expand(N, NQ, D).contiguous()
        qm = self._bool_mask(tgt_query_mask, (NQ, J), dev)
        pm = self._bool_mask(tgt_padding_mask, (N, J), dev)
        cm = self._bool_mask(tgt_mask, (J, J), dev) if self.cfg.dec_depth > 1 else None
        out = torch.empty((N, NQ, D), dtype=torch.float32, device=dev)
        eng.decode(N, J, NQ, ids.data_ptr(), mem.data_ptr(), q.data_ptr() if q is not None else None,
                   qm.data_ptr() if qm is not None else None, pm.data_ptr() if pm is not None else None, out.data_ptr(),
                   torch.cuda.current_stream(dev).cuda_stream, cm.data_ptr() if cm is not None else None)
        return out

    def forward(self, tokenizer: Tokenizer, images: Union[Tensor, List[Any]], max_length: Optional[int] = None,
                return_ids: bool = False, forced_ids: Optional[Tensor] = None,
                forced_refine: Optional[Tensor] = None, *, rotation: Rotation = 0, class_mask: Optional[Tensor] = None):
        """`images`: normalised float [N, 3, H, W], uint8 [N, H, W, 3] at img_size, or a list of raw crops of any size
        (uint8 [h, w, 3] tensors, all CUDA or all CPU, or PIL images in mode RGB) that the engine rotates by `rotation`
        and resizes as the reference's test transform does.  `class_mask`: per-image allowlist words (allowlist_mask)."""
        logits, ids, steps, _ = self._run(images, max_length, self.decode_ar, self.refine_iters, forced_ids, forced_refine,
                                          rotation, class_mask)
        if max_length is None and self.decode_ar and not self.refine_iters:
            # model.py:144-147: with no refinement the reference returns only the S steps it ran
            S = int(steps.item())
            logits, ids = logits[:, :S], ids[:, :S]
        if return_ids:
            return logits, ids
        return logits

    def forward_with_attention(self, images: Union[Tensor, List[Any]], max_length: Optional[int] = None, *,
                               rotation: Rotation = 0, class_mask: Optional[Tensor] = None):
        """forward(tokenizer, images, max_length, return_ids=True) plus the cross-attention maps of the decoder's last
        layer (parseq_forward_args.attn_maps): (logits [N, S, C], ids [N, S], maps fp32 [N, S, T]), maps[b, i] the
        head-averaged weights over the T image tokens of the query that produced logits[b, i].  The logits and ids are
        bit-identical to forward's."""
        logits, ids, steps, maps = self._run(images, max_length, self.decode_ar, self.refine_iters, rotation=rotation,
                                             class_mask=class_mask, attn_maps=True)
        if max_length is None and self.decode_ar and not self.refine_iters:
            S = int(steps.item())
            logits, ids, maps = logits[:, :S], ids[:, :S], maps[:, :S]
        return logits, ids, maps

    def read_oriented(self, crops: List[Any], orientations: Sequence[int] = ORIENTATIONS,
                      min_confidence: Optional[float] = None, max_length: Optional[int] = None, *,
                      class_mask: Optional[Tensor] = None, attn_maps: bool = False):
        """Orientation search (parseq_forward_crops_oriented): each raw crop read at orientations[0] and, unless its
        confidence is >= min_confidence, at the others too, keeping the most confident reading (ties to the earlier
        orientation, NaN last).  (logits [N, S, C], ids [N, S], rotation int64 [N], confidence [N], maps [N, S, T] or
        None); logits and ids as forward returns them, each crop's bit-identical to forward(rotation=rotation[b]) up to
        its EOS."""
        logits, ids, steps, maps, rot, conf = self._run_oriented(crops, orientations, min_confidence, max_length,
                                                                 self.decode_ar, self.refine_iters, class_mask, attn_maps)
        if max_length is None and self.decode_ar and not self.refine_iters:
            S = int(steps.item())
            logits, ids = logits[:, :S], ids[:, :S]
            maps = maps[:, :S] if maps is not None else None
        return logits, ids, rot.long(), conf, maps


class VitstrModel(_EngineModule):
    """Mirror of `strhub.models.vitstr.model.ViTSTR` (vitstr/model.py:14-28): a timm ViT with class token whose head is
    applied per token.  Parameters carry timm's names (`cls_token`, `pos_embed`, `blocks.<i>...`, `norm`, `head`)."""

    def forward_features(self, x: Tensor) -> Tensor:
        return self._features(x)

    def forward_tokens(self, images: Union[Tensor, List[Any]], max_length: Optional[int] = None, return_ids: bool = False,
                       *, rotation: Rotation = 0, class_mask: Optional[Tensor] = None):
        """`self.forward(images, max_length + 2)[:, 1:]` (vitstr/system.py:65-71) in one engine call; `images` and
        `class_mask` as in ParseqModel.forward."""
        logits, ids, _, _ = self._run(images, max_length, False, 0, rotation=rotation, class_mask=class_mask)
        return (logits, ids) if return_ids else logits

    def read_oriented(self, crops: List[Any], orientations: Sequence[int] = ORIENTATIONS,
                      min_confidence: Optional[float] = None, max_length: Optional[int] = None, *,
                      class_mask: Optional[Tensor] = None):
        """ParseqModel.read_oriented over forward_tokens' logits: (logits, ids, rotation int64 [N], confidence [N],
        None)."""
        logits, ids, _, _, rot, conf = self._run_oriented(crops, orientations, min_confidence, max_length, False, 0,
                                                          class_mask)
        return logits, ids, rot.long(), conf, None

    def forward(self, x: Tensor, seqlen: int = 25) -> Tensor:
        raise NotImplementedError(
            "the engine computes head(norm(x))[:, 1:seqlen] only: token 0 (the class token) is discarded by the only "
            "reference caller (vitstr/system.py:68-70); use forward_tokens(images, max_length) or forward_features(x)")


class _HParams(SimpleNamespace):
    def __getitem__(self, k):
        return getattr(self, k)

    def __contains__(self, k):
        return hasattr(self, k)

    def keys(self):
        return self.__dict__.keys()


class _System(nn.Module):
    """The inference-side surface of `strhub.models.base.CrossEntropySystem` (base.py:36-44,112-143,179-207)."""

    # why return_attention is refused, or None where the decoder has cross-attention maps
    _no_attention: Optional[str] = None

    def _check_attention(self, return_attention: bool):
        if return_attention and self._no_attention is not None:
            raise NotImplementedError(self._no_attention)

    def _grid_maps(self, maps: Tensor) -> Tensor:
        """fp32 [..., T] maps as [..., gh, gw] over the patch grid."""
        gh, gw = self.model.cfg.grid
        return maps.view(*maps.shape[:-1], gh, gw)

    def _init_base(self, charset_train, charset_test, batch_size, lr, warmup_pct, weight_decay):
        self.tokenizer = Tokenizer(charset_train)
        self.charset_adapter = CharsetAdapter(charset_test)
        self.bos_id, self.eos_id, self.pad_id = self.tokenizer.bos_id, self.tokenizer.eos_id, self.tokenizer.pad_id
        self.batch_size, self.lr, self.warmup_pct, self.weight_decay = batch_size, lr, warmup_pct, weight_decay

    @property
    def device(self) -> torch.device:
        return self.model._device

    def preprocess(self, crops: Sequence[Any], rotation: Rotation = 0) -> Tensor:
        """The reference's test transform up to the uint8 image (module.py:69-82: rotate, T.Resize(img_size, BICUBIC)) of
        a list of raw crops, on the device: CUDA uint8 [N, H, W, 3], what `forward` takes as a tensor."""
        return self.model.preprocess(crops, rotation)

    def crop_regions(self, frames, regions, frame_index=None) -> RegionCrops:
        """Text regions of full frames (a detector's output), rectified on the device into crops that forward,
        read_oriented, score, beam_search, lexicon_decode, preprocess and locate take as raw crops.
        `frames`: one frame or a list of frames, each a uint8 [H, W, 3] tensor (CUDA or CPU) or an RGB PIL image; CPU
        and PIL frames are uploaded to the model's device.  `regions`, as a tensor, array or list: float corners
        [M, 4, 2] in reading order (TL, TR, BR, BL, frame pixels; pixel i covers [i, i + 1)); integer boxes [M, 4] =
        (x0, y0, x1, y1); polygons of curved text [M, 2k, 2], 3 <= k <= 32; or a list of M point arrays [n_i, 2] that
        mixes quads (n_i = 4) and polygons of different even lengths.  `frame_index`: int [M], the frame of each region
        (required with more than one frame).
        Quads: crop i is w = max(1, round(max(|TR - TL|, |BR - BL|))) by h = max(1, round(max(|BL - TL|, |BR - TR|)))
        pixels (round half up), exactly frame.transform((w, h), PERSPECTIVE, coeffs, BICUBIC) of PIL with the
        closed-form square-to-quad coefficients (parseq_b200/regions.py), 0 outside the frame; a box gives
        frame[y0:y1, x0:x1].
        Polygons are in the Total-Text / CTW1500 order: the top edge p_0..p_{k-1} left to right, then the bottom edge
        q_0..q_{k-1} right to left (FCENet, TextSnake, PAN and ABCNet-style outputs).  A DBNet-style contour has to be
        split into those two edges by the caller.  The crop is as long as the longer edge and as tall as the widest
        p_j - q_{k-1-j} gap (rounded half up) and is rectified by the thin-plate spline of TRBA's GridGenerator with
        the polygon as its fiducial points, then sampled like a quad (include/parseq_b200.h, parseq_warp_polygons).
        ValueError, with the region's index, for non-finite points; degenerate, self-intersecting or non-convex quads;
        polygons of an odd count, fewer than 6 or more than 64 points, or self-intersecting; crop sides over 8192; and
        bad shapes or dtypes.  Returns a RegionCrops: the M CUDA crops, with .quads, .coeffs, .polygons, .tps,
        .frame_index and .to_frame(points, i), which maps points of crop i (such as locate's centres) back into its
        frame, through the thin-plate spline for a polygon."""
        return self.model.crop_regions(frames, regions, frame_index)

    def allowlist_mask(self, allowlist: Allowlist, batch: int) -> Optional[Tensor]:
        """`allowlist` of `forward` as the engine's per-image class mask (module function allowlist_mask)."""
        return allowlist_mask(self.tokenizer, allowlist, batch, self.model.cfg.num_classes)

    def postprocess(self, logits: Tensor):
        """Device-side greedy decode of logits [N, L, C]: (labels, confidences) with the semantics of
        `logits.softmax(-1)` -> `tokenizer.decode` -> `prob.prod()` (base.py:132-142); one small D2H per batch."""
        eng = self.model.engine()
        logits = logits.contiguous()
        N, L, _ = logits.shape
        dev = logits.device
        ids = torch.empty((N, L), dtype=torch.int32, device=dev)
        lengths = torch.empty((N,), dtype=torch.int32, device=dev)
        conf = torch.empty((N,), dtype=torch.float32, device=dev)
        eng.postprocess(logits.data_ptr(), N, L, ids.data_ptr(), lengths.data_ptr(), conf.data_ptr(),
                        torch.cuda.current_stream(dev).cuda_stream, self.eos_id)
        ids_h, len_h, conf_h = ids.cpu().tolist(), lengths.cpu().tolist(), conf.cpu().tolist()
        labels = [self.tokenizer._ids2tok(row[:n], True) for row, n in zip(ids_h, len_h)]
        return labels, conf_h

    def read_oriented(self, crops: List[Any], orientations: Sequence[int] = ORIENTATIONS,
                      min_confidence: Optional[float] = None, max_length: Optional[int] = None,
                      allowlist: Allowlist = None) -> Tuple[Tensor, Tensor, Tensor]:
        """Reads each raw crop the right way up: (logits, rotation int64 [N], confidence fp32 [N]).  Every crop is
        read at orientations[0]; a crop whose confidence (postprocess's) is below `min_confidence`, or every crop when
        it is None, is also read at the other orientations (1 to 4 distinct values of 0, 90, 180, 270, counter-
        clockwise as `rotation`) and keeps the reading of highest confidence: ties go to the earlier orientation, NaN
        ranks below every number.  Each crop's logits are forward(rotation=rotation[b])'s up to its EOS (rows from the
        step count of the pass that produced the reading are 0), and postprocess(logits) returns `confidence` exactly.
        The search runs on the device; with min_confidence the engine synchronises once to list the crops to re-read.
        CUDA crops give CUDA results, CPU crops CPU results."""
        mask = self.allowlist_mask(allowlist, len(crops) if isinstance(crops, (list, tuple)) else crops.shape[0])
        logits, _, rotation, confidence, _ = self.model.read_oriented(crops, orientations, min_confidence, max_length,
                                                                      class_mask=mask)
        return logits, rotation, confidence

    def score(self, images: Union[Tensor, List[Any]], candidates: Candidates, *, rotation: Rotation = 0,
              return_token_logprobs: bool = False, return_attention: bool = False):
        """Log-likelihood of each candidate label for each image: fp32 [N, Kmax], -inf past an image's own candidates.
        PARSeq: sum over i = 0..n of log_softmax(head(decode(...)))[i, t_i] under the canonical left-to-right masks, with
        targets t = (c_1..c_n, EOS) - minus the summed cross-entropy of permutation 0 of the reference's training_step.
        ViTSTR: the same sum over its per-token logits.  `candidates`: one list of strings for every image (a lexicon),
        or one non-empty list per image.  With return_token_logprobs also the terms [N, Kmax, max_label_length + 1]
        (0 past each label's EOS and past an image's candidates).  With return_attention (PARSeq) also the maps fp32
        [N, Kmax, max_label_length + 1, gh, gw]: [b, k, i] is the cross-attention of the decoder's last layer for the
        query that predicts character i of candidate k (i = n: its EOS), in the teacher-forced pass the score comes
        from, averaged over the heads as in read_with_attention; 0 past each label's EOS and past an image's candidates.
        `images` as forward takes them; the result is on the images' device (CPU for CPU crops)."""
        self._check_attention(return_attention)
        N = len(images) if isinstance(images, (list, tuple)) else images.shape[0]
        cfg = self.model.cfg
        targets, lengths, per_image = pack_candidates(self.tokenizer, candidates, N, cfg.max_label_length, cfg.num_classes)
        out = self.model.score(images, targets, lengths, per_image, rotation=rotation,
                               return_token_logprobs=return_token_logprobs, return_attention=return_attention)
        out = out if isinstance(out, tuple) else (out,)
        scores = out[0]
        tlp = out[1] if return_token_logprobs else None
        maps = out[-1] if return_attention else None
        K = int(per_image.max())
        dev = scores.device
        img = torch.repeat_interleave(torch.arange(N), per_image.long())
        col = torch.arange(len(img)) - torch.repeat_interleave(torch.cumsum(per_image.long(), 0) - per_image.long(),
                                                                per_image.long())
        idx = (img * K + col).to(dev)
        grid = torch.full((N * K,), float("-inf"), dtype=torch.float32, device=dev)
        grid[idx] = scores
        if isinstance(images, (list, tuple)) and all(not (isinstance(c, Tensor) and c.is_cuda) for c in images):
            dev = torch.device("cpu")
        grid = grid.view(N, K).to(dev)
        res = (grid,)
        for rows in (tlp, maps):
            if rows is not None:                     # [M, L, ...] -> [N, Kmax, L, ...], zero past an image's candidates
                full = torch.zeros((N * K,) + tuple(rows.shape[1:]), dtype=torch.float32, device=rows.device)
                full[idx] = rows
                res += (full.view((N, K) + tuple(rows.shape[1:])).to(dev),)
        if maps is not None:
            res = res[:-1] + (self._grid_maps(res[-1]),)
        return res if len(res) > 1 else grid

    def compile_lexicon(self, candidates: Candidates) -> Lexicon:
        """A word list (shared by every image) or one list per image, compiled for beam_search(lexicon=) and
        lexicon_decode(beam_width=): checked as score checks candidates, de-duplicated, and built into a prefix trie
        (a forest with one root per distinct per-image list).  Words match charset_train exactly (no case folding).
        Compiling once saves the trie build on every call; the device copy is made once per engine."""
        cfg = self.model.cfg
        return Lexicon(self.tokenizer, candidates, cfg.max_label_length, cfg.num_classes)

    def lexicon_decode(self, images: Union[Tensor, List[Any]], lexicon: Union[Candidates, Lexicon], *,
                       rotation: Rotation = 0, beam_width: Optional[int] = None, return_attention: bool = False):
        """Lexicon-constrained recognition: for each image the candidate the model rates most likely (score), as
        (labels, log_probs).  The pick is torch.argmax of the image's scores: the first maximum, or the first NaN.
        With `beam_width` the pick is the best hypothesis of a lexicon-constrained beam search of that width instead,
        at a cost that does not grow with the lexicon (`lexicon` may then be a compiled Lexicon); an image with no
        reachable word gets label None and -inf.  With return_attention (PARSeq) also the chosen word's maps fp32
        [N, max_label_length + 1, gh, gw], as score returns them (0 for an image with no word)."""
        self._check_attention(return_attention)
        if beam_width is not None:
            out = self.beam_search(images, beam_width, rotation=rotation, lexicon=lexicon,
                                   return_attention=return_attention)
            labels = [h[0] if h else None for h in out[0]]
            return (labels, out[1][:, 0]) + ((out[2][:, 0],) if return_attention else ())
        if isinstance(lexicon, Lexicon):
            raise TypeError("a compiled Lexicon serves the beam search only: pass beam_width, or the word lists to score "
                            "every word")
        out = self.score(images, lexicon, rotation=rotation, return_attention=return_attention)
        scores = out[0] if return_attention else out
        N = scores.shape[0]
        rows = [lexicon] * N if all(isinstance(c, str) for c in lexicon) else list(lexicon)
        best = scores.argmax(-1)
        best_h = best.tolist()
        labels = [rows[b][k] for b, k in enumerate(best_h)]
        res = (labels, scores.gather(1, best[:, None])[:, 0])
        if not return_attention:
            return res
        maps = out[1]
        return res + (maps[torch.arange(N, device=maps.device), best.to(maps.device)],)

    def beam_search(self, images: Union[Tensor, List[Any]], beam_width: int = 5, max_length: Optional[int] = None, *,
                    rotation: Rotation = 0, allowlist: Allowlist = None, lexicon: Union[Candidates, Lexicon, None] = None,
                    return_attention: bool = False):
        """The `beam_width` most likely readings of each image by beam search on the device, as (labels, scores):
        labels[b] lists image b's hypotheses best first (fewer than beam_width when fewer exist), scores is fp32
        [N, beam_width], -inf padded, with each hypothesis's AR log-likelihood (what `score` returns for that label).
        PARSeq runs its AR decoder without refinement, whatever decode_ar / refine_iters say; ViTSTR searches over its
        per-position logits.  With beam_width = 1 the label is the greedy AR reading.  `images` as forward takes them;
        `allowlist` as in forward.  The scores are on the images' device (CPU for CPU crops).
        `lexicon` (a word list for every image, one list per image, or a compiled Lexicon) restricts every hypothesis to
        a word of the image's list that ends with EOS within max_length characters; the log-sum-exp of each step stays
        over all allowed classes, so a score is still `score`'s for that word.  With return_attention (PARSeq) also the
        hypotheses' maps fp32 [N, beam_width, num_steps, gh, gw]: hypothesis k's are `score`'s maps of its label, bit for
        bit, 0 past its EOS and for a missing hypothesis."""
        check_beam_width(beam_width)
        self._check_attention(return_attention)
        N = len(images) if isinstance(images, (list, tuple)) else images.shape[0]
        mask = self.allowlist_mask(allowlist, N)
        roots = None
        if lexicon is not None:
            if not isinstance(lexicon, Lexicon):
                lexicon_rows(lexicon, N)                   # the image count of per-image lists, before the trie build
                lexicon = self.compile_lexicon(lexicon)
            roots = lexicon.roots_for(N)
        out = self.model.beam_search(images, beam_width, max_length, rotation=rotation, class_mask=mask,
                                     lexicon=lexicon, roots=roots, return_attention=return_attention)
        ids, lengths, scores = out[:3]
        ids_h, len_h = ids.cpu().tolist(), lengths.cpu().tolist()
        labels = [[self.tokenizer._ids2tok(ids_h[b][k][:n], True) for k, n in enumerate(len_h[b]) if n >= 0]
                  for b in range(N)]
        maps = self._grid_maps(out[3]) if return_attention else None
        if isinstance(images, (list, tuple)) and all(not (isinstance(c, Tensor) and c.is_cuda) for c in images):
            scores = scores.cpu()
            maps = maps.cpu() if maps is not None else None
        return (labels, scores, maps) if return_attention else (labels, scores)

    # base.py:112-143,179-180 (test path only; validation loss is a training concern)
    def _eval_step(self, batch, validation: bool = False):
        images, labels = batch
        logits = self.forward(images)
        preds, confs = self.postprocess(logits)
        correct = total = label_length = 0
        ned = confidence = 0.0
        for pred, conf_i, gt in zip(preds, confs, labels):
            confidence += conf_i
            pred = self.charset_adapter(pred)
            ned += edit_distance(pred, gt) / max(len(pred), len(gt), 1)
            correct += int(pred == gt)
            total += 1
            label_length += len(pred)
        return dict(output=BatchResult(total, correct, ned, confidence, label_length, None, None))

    def test_step(self, batch, batch_idx):
        return self._eval_step(batch, False)

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path: str, map_location="cpu", **kwargs):
        """Lightning .ckpt layout: {'hyper_parameters': ctor kwargs, 'state_dict': {'model.<key>': tensor}}."""
        ckpt = torch.load(checkpoint_path, map_location=map_location, weights_only=False)
        hp = dict(ckpt.get("hyper_parameters", {}))
        hp.update(kwargs)
        model = cls(**hp)
        sd = {k[len("model."):]: v for k, v in ckpt["state_dict"].items() if k.startswith("model.")}
        model.model.load_state_dict(sd)
        return model


class PARSeq(_System):
    def __init__(self, charset_train: str, charset_test: str, max_label_length: int, batch_size: int = 384,
                 lr: float = 7e-4, warmup_pct: float = 0.075, weight_decay: float = 0.0,
                 img_size: Sequence[int] = (32, 128), patch_size: Sequence[int] = (4, 8), embed_dim: int = 384,
                 enc_num_heads: int = 6, enc_mlp_ratio: int = 4, enc_depth: int = 12, dec_num_heads: int = 12,
                 dec_mlp_ratio: int = 4, dec_depth: int = 1, perm_num: int = 6, perm_forward: bool = True,
                 perm_mirrored: bool = True, decode_ar: bool = True, refine_iters: int = 1, dropout: float = 0.1,
                 **kwargs: Any) -> None:
        super().__init__()
        hp = dict(charset_train=charset_train, charset_test=charset_test, max_label_length=max_label_length,
                  batch_size=batch_size, lr=lr, warmup_pct=warmup_pct, weight_decay=weight_decay,
                  img_size=list(img_size), patch_size=list(patch_size), embed_dim=embed_dim,
                  enc_num_heads=enc_num_heads, enc_mlp_ratio=enc_mlp_ratio, enc_depth=enc_depth,
                  dec_num_heads=dec_num_heads, dec_mlp_ratio=dec_mlp_ratio, dec_depth=dec_depth, perm_num=perm_num,
                  perm_forward=perm_forward, perm_mirrored=perm_mirrored, decode_ar=decode_ar,
                  refine_iters=refine_iters, dropout=dropout)
        hp.update(kwargs)
        self.hparams = _HParams(**hp)
        self._init_base(charset_train, charset_test, batch_size, lr, warmup_pct, weight_decay)
        cfg = ParseqConfig(charset_train=charset_train, charset_test=charset_test, max_label_length=max_label_length,
                           img_size=tuple(img_size), patch_size=tuple(patch_size), embed_dim=embed_dim,
                           enc_num_heads=enc_num_heads, enc_mlp_ratio=enc_mlp_ratio, enc_depth=enc_depth,
                           dec_num_heads=dec_num_heads, dec_mlp_ratio=dec_mlp_ratio, dec_depth=dec_depth,
                           decode_ar=decode_ar, refine_iters=refine_iters, dropout=dropout,
                           name=str(kwargs.get("name", "parseq")))
        try:
            self.model = ParseqModel(cfg)
        except EngineError as e:  # pragma: no cover
            raise InvalidModelError(str(e)) from e

    def forward(self, images: Union[Tensor, List[Any]], max_length: Optional[int] = None, *, rotation: Rotation = 0,
                allowlist: Allowlist = None) -> Tensor:
        """`images`: a tensor, as the reference takes, or a list of raw crops of any size (ParseqModel.forward).
        `allowlist`: None, one string for every image, or one Optional[str] per image: the characters each image may
        decode to.  Every greedy decision (AR loop, refinement, NAR) is constrained on the device, as if the reference's
        head returned -inf for every other character; those logits come back as -inf."""
        mask = self.allowlist_mask(allowlist, len(images) if isinstance(images, (list, tuple)) else images.shape[0])
        return self.model.forward(self.tokenizer, images, max_length, rotation=rotation, class_mask=mask)

    def read_with_attention(self, images: Union[Tensor, List[Any]], max_length: Optional[int] = None, *,
                            rotation: Rotation = 0, allowlist: Allowlist = None) -> Tuple[Tensor, Tensor]:
        """`forward` plus where the decoder looked: (logits, maps) with logits exactly forward's and maps fp32
        [N, S, gh, gw] (S = logits.shape[1], (gh, gw) the patch grid): maps[b, i] is the cross-attention of the decoder's
        last layer for the query that produced logits[b, i], averaged over the heads as nn.MultiheadAttention averages
        them, from the last refinement pass, the NAR pass, or AR step i when there is no refinement.  Each map sums to
        1 over the grid.  Inputs and result devices as in forward."""
        mask = self.allowlist_mask(allowlist, len(images) if isinstance(images, (list, tuple)) else images.shape[0])
        logits, _, maps = self.model.forward_with_attention(images, max_length, rotation=rotation, class_mask=mask)
        gh, gw = self.model.cfg.grid
        return logits, maps.view(maps.shape[0], maps.shape[1], gh, gw)

    def locate(self, images: Union[Tensor, List[Any]], max_length: Optional[int] = None, *, rotation: Rotation = 0,
               allowlist: Allowlist = None, threshold: float = 0.5, orientations: Optional[Sequence[int]] = None,
               min_confidence: Optional[float] = None, text: Union[None, str, Sequence[str]] = None):
        """Where each character was read: (labels, confidences, centers, boxes).  labels / confidences are postprocess's
        of the forward logits; centers[b] fp32 [n_b, 2] = (x, y) and boxes[b] fp32 [n_b, 4] = (x0, y0, x1, y1), one row
        per character of labels[b], from its map of read_with_attention: the map-weighted centroid of the patch-cell
        centres, and the extent of the cells whose weight is >= threshold * the map's maximum.  Coordinates are pixels of
        the input: of the img_size image for tensors, of each original crop for raw crops (the resize scale and each
        crop's rotation undone).  Results on the device of the outputs, as forward returns them.  With `orientations`
        (raw crops only) each crop is read in the orientation read_oriented chooses, and its points are mapped back
        under that rotation.
        With `text` (one string for every image, or one per image) the characters located are those of the given text
        rather than of the model's reading (forced alignment): (labels = the texts, log-likelihoods fp32 [N] as score
        gives them, centers, boxes), each character's map the one score(return_attention=True) gives it.  The text's
        characters must be in charset_train (ValueError otherwise, as in score); it takes the place of max_length,
        allowlist and orientations."""
        if text is not None:
            if max_length is not None or allowlist is not None or orientations is not None or min_confidence is not None:
                raise ValueError("text fixes the characters to locate: it cannot be combined with max_length, "
                                 "allowlist, orientations or min_confidence")
            N = len(images) if isinstance(images, (list, tuple)) else images.shape[0]
            if isinstance(text, str):
                texts = [text] * N
            elif isinstance(text, (list, tuple)) and len(text) == N and all(isinstance(t, str) for t in text):
                texts = list(text)
            else:
                raise ValueError(f"text must be one string or a list of {N} strings (one per image)")
            scores, maps = self.score(images, [[t] for t in texts], rotation=rotation, return_attention=True)
            centers, boxes = self._locate_maps(images, maps[:, 0], [len(t) for t in texts], rotation, threshold)
            return texts, scores[:, 0], centers, boxes
        if orientations is None:
            if min_confidence is not None:
                raise ValueError("min_confidence needs orientations")
            logits, maps = self.read_with_attention(images, max_length, rotation=rotation, allowlist=allowlist)
        else:
            if _is_rotation_list(rotation) or rotation:
                raise ValueError("rotation and orientations cannot be combined: the search chooses each crop's rotation")
            mask = self.allowlist_mask(allowlist, len(images) if isinstance(images, (list, tuple)) else images.shape[0])
            logits, _, rot, _, maps = self.model.read_oriented(images, orientations, min_confidence, max_length,
                                                               class_mask=mask, attn_maps=True)
            gh, gw = self.model.cfg.grid
            maps = maps.view(maps.shape[0], maps.shape[1], gh, gw)
            rotation = rot.tolist()
        labels, confs = self.postprocess(logits.to(self.device))
        centers, boxes = self._locate_maps(images, maps, [len(label) for label in labels], rotation, threshold)
        return labels, confs, centers, boxes

    def _locate_maps(self, images, maps: Tensor, counts: Sequence[int], rotation: Rotation, threshold: float):
        """(centers, boxes) of the first counts[b] maps of each image (maps [N, S, gh, gw]) as locate returns them: in
        pixels of the img_size image for tensors, of each original crop for raw crops (its resize and rotation undone)."""
        cfg = self.model.cfg
        crops = isinstance(images, (list, tuple))
        centers: List[Tensor] = []
        boxes: List[Tensor] = []
        for b, n in enumerate(counts):
            c, bx = attention_centers_boxes(maps[b, :n], cfg.patch_size, threshold)
            if crops:
                hw = _crop_hw(images[b])
                c = unrotate_points(c, hw, cfg.img_size, _rotation_of(rotation, b))
                bx = unrotate_boxes(bx, hw, cfg.img_size, _rotation_of(rotation, b))
            centers.append(c)
            boxes.append(bx)
        return centers, boxes


class ViTSTR(_System):
    """Mirror of `strhub.models.vitstr.system.ViTSTR` (vitstr/system.py:29-71), inference side."""

    _no_attention = ("ViTSTR has no decoder cross-attention: its characters are read from the encoder's own tokens, so "
                     "there are no per-character maps to return")

    def __init__(self, charset_train: str, charset_test: str, max_label_length: int, batch_size: int = 384,
                 lr: float = 8.9e-4, warmup_pct: float = 0.075, weight_decay: float = 0.0,
                 img_size: Sequence[int] = (224, 224), patch_size: Sequence[int] = (16, 16), embed_dim: int = 384,
                 num_heads: int = 6, **kwargs: Any) -> None:
        super().__init__()
        hp = dict(charset_train=charset_train, charset_test=charset_test, max_label_length=max_label_length,
                  batch_size=batch_size, lr=lr, warmup_pct=warmup_pct, weight_decay=weight_decay,
                  img_size=list(img_size), patch_size=list(patch_size), embed_dim=embed_dim, num_heads=num_heads)
        hp.update(kwargs)
        self.hparams = _HParams(**hp)
        self._init_base(charset_train, charset_test, batch_size, lr, warmup_pct, weight_decay)
        self.max_label_length = max_label_length
        # depth=12, mlp_ratio=4, qkv_bias=True are fixed by the reference ctor (vitstr/system.py:50-59)
        cfg = ParseqConfig(charset_train=charset_train, charset_test=charset_test, max_label_length=max_label_length,
                           img_size=tuple(img_size), patch_size=tuple(patch_size), embed_dim=embed_dim,
                           enc_num_heads=num_heads, enc_mlp_ratio=4, enc_depth=12, arch="vitstr",
                           name=str(kwargs.get("name", "vitstr")))
        try:
            self.model = VitstrModel(cfg)
        except EngineError as e:  # pragma: no cover
            raise InvalidModelError(str(e)) from e

    def forward(self, images: Union[Tensor, List[Any]], max_length: Optional[int] = None, *, rotation: Rotation = 0,
                allowlist: Allowlist = None) -> Tensor:
        """`allowlist` as in PARSeq.forward: it constrains the argmax of every token position."""
        mask = self.allowlist_mask(allowlist, len(images) if isinstance(images, (list, tuple)) else images.shape[0])
        return self.model.forward_tokens(images, max_length, rotation=rotation, class_mask=mask)

    def read_with_attention(self, *args, **kwargs):
        raise NotImplementedError("ViTSTR has no decoder cross-attention: its characters are read from the encoder's "
                                  "own tokens, so there are no per-character maps to return")

    def locate(self, *args, **kwargs):
        raise NotImplementedError("ViTSTR has no decoder cross-attention, so characters cannot be located from it")

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path: str, map_location="cpu", **kwargs):
        return super().load_from_checkpoint(checkpoint_path, map_location, **kwargs)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        """Released ViTSTR weights are saved from the SYSTEM (strhub/models/utils.py:80-82: `m = model`), i.e. with a
        'model.' prefix; accept both layouts."""
        if all(k.startswith("model.") for k in state_dict):
            state_dict = {k[len("model."):]: v for k, v in state_dict.items()}
        return self.model.load_state_dict(state_dict, strict=strict, **kw)
