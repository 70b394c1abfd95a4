"""CPU reference of the beam-selection building blocks (kernels.cuh beam_select_kernel, gemm.cuh gemm_topk_epilogue /
gemm_lse_epilogue, lse_merge), for tests/test_gpu_selection_kernels.py and tests/test_selection_reference_cpu.py.

- `beam_order_key` / `key_value` / `key_class`: the 64-bit expansion order of a (logit, class) pair in numpy.
- `tile_partials`: per 128-column tile (max, sum of exp(v - max)) in fp64 over the allowed classes.
- Gapped rows: among its allowed classes a row has a unique maximum m, every other allowed finite logit is an integer
  <= m - 128, and every value is a multiple of 128 of magnitude <= 2^15 (so bf16-exact).  Then exp(v - m) underflows to
  0 in fp32 for every other class, the fp32 log-sum-exp is exactly m, every term v - m is an integer, and an fp32 beam
  search matches the fp64 oracle (beam_oracle / lexicon_oracle) bit for bit.  `emulate_*` replay the kernels' fp32
  summation orders so that the claim can be checked without a GPU.
- `gapped_logits_fn` / `bf16_logits_fn`: prefix-dependent logits_fn's in beam_oracle's convention.
"""
from __future__ import annotations

import zlib
from typing import Optional, Sequence

import numpy as np

TILE = 128
TOPK_LD = 16
GAP = 128
VMAX = 1 << 15


# ---------------------------------------------------------------- keys
def beam_order_key(x, c) -> np.ndarray:
    """ptx.cuh beam_order_key over arrays: larger = earlier; NaN first, then the logit descending, ties to the lower
    class; -0 counts as +0.  The caller leaves -inf and masked classes out (key 0 = none)."""
    x = np.asarray(x, dtype=np.float32)
    c = np.asarray(c, dtype=np.int64)
    x = np.where(x == 0, np.float32(0), x)
    u = x.view(np.uint32).astype(np.uint64)
    o = np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000)
    o = np.where(np.isnan(x), np.uint64(0xffffffff), o).astype(np.uint64)
    return (o << np.uint64(32)) | (np.uint64(0xffffffff) - c.astype(np.uint64))


def key_value(key) -> np.ndarray:
    """The logit of a key (NaN for a NaN key; -0 comes back as +0)."""
    key = np.asarray(key, dtype=np.uint64)
    o = (key >> np.uint64(32)).astype(np.uint64)
    u = np.where(o & 0x80000000, o & 0x7fffffff, ~o & 0xffffffff).astype(np.uint32)
    v = u.view(np.float32)
    return np.where(o == 0xffffffff, np.float32(np.nan), v)


def key_class(key) -> np.ndarray:
    key = np.asarray(key, dtype=np.uint64)
    return (np.uint64(0xffffffff) - (key & np.uint64(0xffffffff))).astype(np.int64)


def row_keys(row, allowed=None) -> np.ndarray:
    """The row's expandable classes as keys in expansion order (descending)."""
    row = np.asarray(row, dtype=np.float32)
    ok = row != -np.inf
    if allowed is not None:
        ok &= np.asarray(allowed, dtype=bool)
    c = np.nonzero(ok)[0]
    return np.sort(beam_order_key(row[c], c))[::-1]


# ---------------------------------------------------------------- masks
def mask_words(allowed: Optional[Sequence[bool]], C: int) -> np.ndarray:
    """Allowlist words (parseq_forward_args.class_mask) of one row; EOS is always allowed by the kernels."""
    words = np.zeros((C + 31) // 32, dtype=np.uint32)
    a = np.ones(C, dtype=bool) if allowed is None else np.asarray(allowed, dtype=bool)
    for c in np.nonzero(a)[0]:
        words[c >> 5] |= np.uint32(1 << (c & 31))
    return words


def effective(allowed: Optional[Sequence[bool]], C: int) -> np.ndarray:
    a = np.ones(C, dtype=bool) if allowed is None else np.array(allowed, dtype=bool)
    a[0] = True
    return a


# ---------------------------------------------------------------- fp64 partials
def tile_partials(v, allowed=None):
    """v [M, N] (fp64 logits), allowed [M, N] bool or None -> (mx [M, T], s [M, T]) per 128-column tile in fp64: mx the
    largest allowed non-NaN value (-inf if none), s = sum of exp(v - mx) (exp(v) when mx = -inf); NaN when an allowed value
    is NaN or mx = +inf, as the epilogues give."""
    v = np.asarray(v, dtype=np.float64)
    M, N = v.shape
    T = (N + TILE - 1) // TILE
    ok = np.ones_like(v, dtype=bool) if allowed is None else np.asarray(allowed, dtype=bool)
    w = np.where(ok, v, -np.inf)
    pad = np.full((M, T * TILE), -np.inf)
    pad[:, :N] = w
    pad = pad.reshape(M, T, TILE)
    mx = np.max(np.where(np.isnan(pad), -np.inf, pad), axis=2)
    base = np.where(mx == -np.inf, 0.0, mx)
    with np.errstate(invalid="ignore", over="ignore"):
        s = np.exp(pad - base[:, :, None]).sum(axis=2)
    s = np.where(np.isnan(pad).any(axis=2) | (mx == np.inf), np.nan, s)
    return mx, s


def topk_keys(v, allowed, k: int) -> np.ndarray:
    """[M, T, 16] uint64: per row and tile the k best allowed non--inf classes' keys, 0 after the last."""
    v = np.asarray(v, dtype=np.float32)
    M, N = v.shape
    T = (N + TILE - 1) // TILE
    ok = v != -np.inf
    if allowed is not None:
        ok &= np.asarray(allowed, dtype=bool)
    keys = np.where(ok, beam_order_key(v, np.arange(N)[None, :]), np.uint64(0)).astype(np.uint64)
    pad = np.zeros((M, T * TILE), dtype=np.uint64)
    pad[:, :N] = keys
    best = np.sort(pad.reshape(M, T, TILE), axis=2)[:, :, ::-1][:, :, :k]
    out = np.zeros((M, T, TOPK_LD), dtype=np.uint64)
    out[:, :, :k] = best
    return out


# ---------------------------------------------------------------- float32 emulation of the kernels' LSE
def _f32(x):
    return np.float32(x)


def emulate_lse_row(row, allowed=None) -> np.float32:
    """beam_select_kernel at <= 128 classes (and every lexicon step): lane l takes classes l, l + 32, ..., max and sum
    in that order, then a 16/8/4/2/1 xor butterfly; LSE = m + logf(s)."""
    row = np.asarray(row, dtype=np.float32)
    C = row.shape[0]
    ok = effective(allowed, C)
    m = np.full(32, -np.inf, dtype=np.float32)
    for c in range(C):
        if ok[c]:
            m[c % 32] = np.fmax(m[c % 32], row[c])
    for o in (16, 8, 4, 2, 1):
        m = np.fmax(m, m[np.arange(32) ^ o])
    base = _f32(0) if m[0] == -np.inf else m[0]
    s = np.zeros(32, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for c in range(C):
            if ok[c]:
                s[c % 32] = _f32(s[c % 32] + np.exp(_f32(row[c] - base), dtype=np.float32))
        for o in (16, 8, 4, 2, 1):
            s = (s + s[np.arange(32) ^ o]).astype(np.float32)
        return _f32(m[0] + np.log(s[0], dtype=np.float32))


def emulate_tile_partial(vals, ok) -> tuple:
    """gemm_*_epilogue for one row of one tile (vals [<=128] fp32, ok allowed): quad lane q holds columns i * 8 + 2q + e
    (i < 16, e < 2) in that order; max and sum per lane, then xor 1 and xor 2."""
    v = np.full(TILE, -np.inf, dtype=np.float32)
    v[:len(vals)] = np.where(ok, vals, -np.inf)
    lanes = [[i * 8 + 2 * q + e for i in range(16) for e in range(2)] for q in range(4)]
    mx = np.array([np.fmax.reduce(v[c]) for c in lanes], dtype=np.float32)
    mx = np.fmax(mx, mx[[1, 0, 3, 2]])
    mx = np.fmax(mx, mx[[2, 3, 0, 1]])
    base = _f32(0) if mx[0] == -np.inf else mx[0]
    s = np.zeros(4, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for q in range(4):
            for c in lanes[q]:
                s[q] = _f32(s[q] + np.exp(_f32(v[c] - base), dtype=np.float32))
        s = (s + s[[1, 0, 3, 2]]).astype(np.float32)
        s = (s + s[[2, 3, 0, 1]]).astype(np.float32)
    return mx[0], s[0]


def emulate_lse_tiles(row, allowed=None) -> np.float32:
    """The top-K / LSE epilogues' tile partials merged by lse_merge in column order: M + logf(S)."""
    row = np.asarray(row, dtype=np.float32)
    C = row.shape[0]
    ok = effective(allowed, C)
    parts = [emulate_tile_partial(row[t:t + TILE], ok[t:t + TILE]) for t in range(0, C, TILE)]
    M = np.float32(-np.inf)
    for m, _ in parts:
        M = np.fmax(M, m)
    S = np.float32(0)
    with np.errstate(invalid="ignore", over="ignore"):
        for m, s in parts:
            S = _f32(S + _f32(s * np.exp(_f32(m - M), dtype=np.float32)))
        return _f32(M + np.log(S, dtype=np.float32))


# ---------------------------------------------------------------- gapped rows
def check_gapped(row, allowed=None) -> float:
    """Asserts the gap condition of `row` under `allowed`; returns its allowed maximum m."""
    row = np.asarray(row, dtype=np.float64)
    ok = effective(allowed, row.shape[0])
    fin = row[np.isfinite(row)]
    assert np.all(fin == np.round(fin)) and np.all(np.abs(fin) <= VMAX)
    a = row[ok]
    m = a.max()
    assert np.isfinite(m) and np.count_nonzero(a == m) == 1, "the allowed maximum must be unique"
    rest = a[a != m]
    assert np.all((rest == -np.inf) | (rest <= m - GAP))
    return float(m)


def gapped_row(rng, C: int, allowed=None, neg_inf: float = 0.1, levels: int = 4, top=None) -> np.ndarray:
    """A gapped row: values 128 * integer; the allowed maximum sits at a random allowed class (or `top`), every other
    allowed class `levels` or fewer steps of 128 below it (ties between them are the rule), about `neg_inf` of them -inf;
    masked classes take any multiple of 128, above the maximum too."""
    ok = effective(allowed, C)
    a = int(rng.integers(-40, 41))
    row = (a - rng.integers(1, levels + 1, C)).astype(np.float64) * GAP
    row[rng.random(C) < neg_inf] = -np.inf
    masked = np.nonzero(~ok)[0]
    row[masked] = (a + rng.integers(-3, 4, masked.shape[0])) * GAP
    cand = np.nonzero(ok)[0]
    t = int(rng.choice(cand)) if top is None else int(top)
    row[t] = a * GAP
    check_gapped(row, allowed)
    return row


def _seed(seed, prefix) -> int:
    return zlib.crc32(np.asarray([seed] + list(prefix), dtype=np.int64).tobytes())


class gapped_logits_fn:
    """logits_fn(prefixes) -> rows, a gapped row per prefix (per position when `by_position`: ViTSTR).  `allowed` is the
    image's allowlist (the gap is asserted over it).  With nonfinite > 0 that fraction of rows also gets a NaN or a +inf
    at an allowed class (the row is then not gapped: its LSE is NaN)."""

    def __init__(self, C, seed, allowed=None, by_position=False, nonfinite=0.0, levels=4, neg_inf=0.1):
        self.C, self.seed, self.allowed, self.by_position = C, seed, allowed, by_position
        self.nonfinite, self.levels, self.neg_inf = nonfinite, levels, neg_inf
        self.cache = {}

    def row(self, prefix) -> np.ndarray:
        key = (len(prefix),) if self.by_position else tuple(prefix)
        if key not in self.cache:
            rng = np.random.default_rng(_seed(self.seed, key))
            r = gapped_row(rng, self.C, self.allowed, self.neg_inf, self.levels)
            if self.nonfinite > 0 and rng.random() < self.nonfinite:
                ok = np.nonzero(effective(self.allowed, self.C))[0]
                for c in rng.choice(ok, size=min(2, ok.shape[0]), replace=False):
                    r[c] = np.nan if rng.random() < 0.5 else np.inf
            self.cache[key] = r
        return self.cache[key]

    def __call__(self, prefixes):
        return [self.row(p) for p in prefixes]


class bf16_logits_fn:
    """Random normal logits (scale 3) rounded to bf16: exact in fp32, with exact ties among them."""

    def __init__(self, C, seed, by_position=False):
        self.C, self.seed, self.by_position = C, seed, by_position
        self.cache = {}

    def row(self, prefix) -> np.ndarray:
        key = (len(prefix),) if self.by_position else tuple(prefix)
        if key not in self.cache:
            rng = np.random.default_rng(_seed(self.seed, key))
            self.cache[key] = to_bf16(rng.standard_normal(self.C) * 3.0).astype(np.float64)
        return self.cache[key]

    def __call__(self, prefixes):
        return [self.row(p) for p in prefixes]


def to_bf16(x) -> np.ndarray:
    """Round-to-nearest-even to bf16, returned as float32."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7fff + ((u >> 16) & 1)) & 0xffff0000
    return u.astype(np.uint32).view(np.float32)


# ---------------------------------------------------------------- the cases the GPU tests search (shared with the CPU check)
# (C, K, num_steps, layout, seed): gapped searches driven through parseq_beam_select
SEARCH_CASES = [
    (3, 1, 26, "parseq", 1), (3, 16, 2, "parseq", 2), (95, 2, 26, "parseq", 3), (95, 8, 64, "parseq", 4),
    (128, 3, 26, "parseq", 5), (128, 16, 1, "parseq", 6), (129, 8, 26, "parseq", 7), (129, 16, 2, "parseq", 8),
    (3001, 5, 26, "parseq", 9), (3001, 16, 2, "parseq", 10), (95, 8, 26, "vitstr", 11), (129, 3, 64, "vitstr", 12),
    (3001, 16, 26, "vitstr", 13), (3, 3, 26, "vitstr", 14),
]


def case_allowlists(C: int, seed: int):
    """Per-image allowlists of a search case: none, a random half, the empty allowlist (EOS only), and one that masks
    class 1 and allows the classes across the 31/32 and 127/128 word and tile boundaries."""
    rng = np.random.default_rng(seed + 1000)
    half = rng.random(C) < 0.5
    half[0] = True
    empty = np.zeros(C, dtype=bool)
    empty[0] = True
    edge = np.zeros(C, dtype=bool)
    edge[[c for c in (0, 2, 31, 32, 63, 64, 127, 128, C - 1) if c < C]] = True
    edge[1] = False
    edge[0] = True
    return [None, half, empty, edge]


E2E_CLASSES = (95, 128, 129, 3001, 16384)


def e2e_bias(C: int, seed: int = 0):
    """The head bias of the end-to-end tests (head.weight = 0, so every logits row is this bias) and four per-image
    allowlists.  The maximum is class 5 at 0, a unique runner-up class 9 at -128, then levels -256 and -384 shared by
    many classes, EOS among them at -256, and some -inf classes.  Allowlists: none, a random half holding class 5, one
    that masks class 5 (the runner-up becomes the unique maximum), and the empty allowlist."""
    rng = np.random.default_rng(seed + C)
    bias = -GAP * rng.integers(2, 4, C).astype(np.float64)
    bias[rng.random(C) < 0.1] = -np.inf
    bias[0] = -2 * GAP
    bias[5], bias[9] = 0.0, -GAP
    half = rng.random(C) < 0.5
    half[[0, 5]] = True
    no_top = np.ones(C, dtype=bool)
    no_top[5] = False
    empty = np.zeros(C, dtype=bool)
    empty[0] = True
    allows = [None, half, no_top, empty]
    for a in allows:
        check_gapped(bias, a)
    return bias, allows


def case_logits_fns(C, seed, layout, nonfinite=0.0):
    return [gapped_logits_fn(C, seed * 10 + b, None if a is None else a, layout == "vitstr", nonfinite)
            for b, a in enumerate(case_allowlists(C, seed))]
