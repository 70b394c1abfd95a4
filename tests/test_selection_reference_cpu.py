"""CPU: the numpy beam order of tests/selection_reference.py is beam_oracle's row order; a float32 replay of the kernels'
summation orders (beam_select_kernel's lane-strided row scan, the GEMM epilogues' quad lanes and lse_merge) gives exactly
the fp64 log-sum-exp on every gapped row the GPU selection tests search, which is what lets those tests demand bit
equality; and the ctypes mirror of parseq_beam_select_args matches the header."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import beam_oracle as BO
import selection_reference as SR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exp_and_log_identities_the_exactness_argument_uses():
    assert np.exp(np.float32(0), dtype=np.float32) == 1 and np.log(np.float32(1), dtype=np.float32) == 0
    assert np.exp(np.float32(-SR.GAP), dtype=np.float32) == 0              # underflows in fp32
    assert 1.0 + math.exp(-SR.GAP) == 1.0                                  # and is lost next to 1 in fp64
    assert np.float32(128 * math.exp(-SR.GAP)) * np.exp(np.float32(-SR.GAP), dtype=np.float32) == 0


@pytest.mark.parametrize("seed", range(6))
def test_numpy_key_order_is_the_oracle_row_order(seed):
    rng = np.random.default_rng(seed)
    C = int(rng.integers(2, 300))
    row = rng.integers(-3, 4, C).astype(np.float32)                      # many exact ties
    special = rng.choice(C, size=min(C, 12), replace=False)
    for i, c in enumerate(special):
        row[c] = [np.nan, np.inf, -np.inf, -0.0, 0.0, np.nan][i % 6]
    allowed = rng.random(C) < 0.8
    for a in (None, allowed):
        keys = SR.row_keys(row, a)
        assert SR.key_class(keys).tolist() == BO.row_order(row.astype(np.float64).tolist(), a)
        v = SR.key_value(keys)
        cls = SR.key_class(keys)
        same = np.where(np.isnan(row[cls]), np.isnan(v), v == row[cls])
        assert bool(same.all())
        assert len(set(keys.tolist())) == len(keys)


def test_key_bits_of_hand_picked_values():
    k = SR.beam_order_key(np.array([np.nan, 1.0, 1.0, 0.0, -0.0, -1.0], dtype=np.float32), np.array([7, 2, 3, 4, 3, 0]))
    assert k[0] > k[1] > k[2] > k[4] > k[3] > k[5]                      # -0 ties with +0, the lower class first
    assert SR.key_value(k[4]) == 0 and not np.signbit(SR.key_value(k[4]))
    assert SR.key_class(k).tolist() == [7, 2, 3, 4, 3, 0]


def test_tile_partials_of_hand_made_rows():
    v = np.full((3, 200), -np.inf)
    v[0, 5], v[0, 130] = 2.0, 1.0
    v[1, 7] = np.nan
    v[2, 150] = np.inf
    mx, s = SR.tile_partials(v)
    assert mx[0].tolist() == [2.0, 1.0] and s[0].tolist() == [1.0, 1.0]
    assert mx[1, 0] == -np.inf and np.isnan(s[1, 0]) and (mx[1, 1], s[1, 1]) == (-np.inf, 0.0)
    assert mx[2, 1] == np.inf and np.isnan(s[2, 1])


def _rows_of_case(C, K, S, layout, seed):
    """Every row beam_oracle reads in a search case, with its image's allowlist."""
    out = []
    for fn, a in zip(SR.case_logits_fns(C, seed, layout), SR.case_allowlists(C, seed)):
        BO.beam_search(fn, K, S, a)
        out += [(r, a) for r in fn.cache.values()]
    return out


@pytest.mark.parametrize("case", SR.SEARCH_CASES, ids=lambda c: f"C{c[0]}-K{c[1]}-S{c[2]}-{c[3]}")
def test_float32_replay_gives_the_fp64_lse_on_every_gapped_row(case):
    C, K, S, layout, seed = case
    rows = _rows_of_case(C, K, S, layout, seed)
    assert rows
    for row, a in rows:
        m = SR.check_gapped(row, a)
        ref = BO._lse([row[c] for c in range(C) if SR.effective(a, C)[c]])
        assert ref == m
        assert SR.emulate_lse_row(row.astype(np.float32), a) == np.float32(m)
        if C > SR.TILE:
            assert SR.emulate_lse_tiles(row.astype(np.float32), a) == np.float32(m)


def test_float32_replay_on_end_to_end_bias_rows():
    for C in SR.E2E_CLASSES:
        bias, allows = SR.e2e_bias(C)
        for a in allows:
            m = SR.check_gapped(bias, a)
            assert SR.emulate_lse_row(bias.astype(np.float32), a) == np.float32(m)
            assert SR.emulate_lse_tiles(bias.astype(np.float32), a) == np.float32(m)


def test_gapped_generator_rejects_a_tied_or_shallow_maximum():
    row = np.array([0.0, -128.0, -256.0, -np.inf])
    assert SR.check_gapped(row) == 0.0
    with pytest.raises(AssertionError):
        SR.check_gapped(np.array([0.0, 0.0, -256.0]))
    with pytest.raises(AssertionError):
        SR.check_gapped(np.array([0.0, -127.0, -256.0]))
    # a masked class above the maximum is fine; an allowed one is not
    assert SR.check_gapped(np.array([0.0, 512.0, -128.0]), [True, False, True]) == 0.0


def test_beam_select_args_mirror_the_header():
    from parseq_b200.engine import BeamSelectArgsC
    hdr = open(os.path.join(ROOT, "include", "parseq_b200.h")).read()
    body = re.search(r"typedef struct parseq_beam_select_args \{(.*?)\} parseq_beam_select_args;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        m = re.match(r"(?:const\s+)?(\w+)\s*(\*?)\s*(.*)", decl)
        ctype, ptr, names = m.group(1), m.group(2), m.group(3)
        for n in names.split(","):
            n = n.strip()
            fields.append((n.lstrip("*"), "ptr" if (ptr or n.startswith("*")) else ctype))
    mine = [(n, "ptr" if t is C.c_void_p else {C.c_int32: "int32_t", C.c_int64: "int64_t"}[t])
            for n, t in BeamSelectArgsC._fields_]
    assert mine == fields
    # natural alignment on LP64: the int64 strides after ntiles start on an 8-byte boundary, as in C
    assert BeamSelectArgsC.row0.offset == 32 and C.sizeof(BeamSelectArgsC) % 8 == 0
