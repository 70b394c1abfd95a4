"""Where the cross-attention maps' error budget comes from (no GPU).

As tests/test_decoder_budget_cpu.py does for the logits: for PARSeq-Ti, PARSeq-S and PARSeq-S at depth 2, with sharp (x4)
attention weights and a memory from the oracle's encoder (depth 2), the fp64 maps of tests/attn_maps_reference.py are
compared, schedule by schedule, with
  * the fp32 stand-in (same rounding points, fp32 arithmetic), what a correct implementation looks like: it must stay
    within half of every bound of attn_maps_reference.BOUNDS;
  * each injected bug of attn_maps_reference.BUGS: it must exceed some bound by 2x or more in the schedule it concerns,
    of BOUNDS and of the wider GOLDEN_BOUNDS the engine is held to against the reference's goldens.
So the bounds tests/test_gpu_attn_maps.py holds the engine to sit at least 2x above the stand-in's noise and at least 2x
below each of these mistakes."""
import functools

import pytest
import torch

from attn_maps_reference import BOUNDS, BUGS, GOLDEN_BOUNDS, MapsReference, excess, format_stats, map_stats
from decoder_reference import forced_ar_ids, refine_context

EXPERIMENT = {192: "parseq-tiny", 384: "parseq"}
CASES = [(192, 1), (384, 1), (384, 2)]
B, L = 8, 26
# the schedule each bug is about (the others are checked where they apply: layer0 needs depth >= 2)
BUG_SCHEDULES = {"head0": ("ar", "nar", "refine"), "first_refine": ("refine",), "layer0": ("ar", "nar", "refine"),
                 "no_scale": ("ar", "nar", "refine"), "key_shift": ("ar", "nar", "refine"),
                 "col_major": ("ar", "nar", "refine"), "ar_from_nar": ("ar",)}


@functools.lru_cache(maxsize=None)
def _case(key):
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.config import make_config
    from parseq_b200.weights import init_state_dict, synth_images
    D, depth = key
    cfg = make_config(EXPERIMENT[D], enc_depth=2, dec_depth=depth)
    sd = init_state_dict(cfg, 3, sharp=4.0)
    enc = make_config(EXPERIMENT[D], enc_depth=2)
    mem = ParseqOracle(enc, init_state_dict(enc, 3, sharp=4.0), "fp32").encode(synth_images(cfg, B, 7))
    mem = mem.to(torch.bfloat16).float()
    bos, C = cfg.num_tokens - 2, cfg.num_classes
    ids = forced_ar_ids(B, L, C, bos, 1)[:, 1:]
    ids = torch.cat([ids, torch.zeros((B, 1), dtype=ids.dtype)], dim=1)      # the returned ids [B, L]
    ctxs = (refine_context(B, L, C, bos, [1, 5, 12, 20, 25, None], 2), refine_context(B, L, C, bos, [3, 9, None], 4))
    return cfg, sd, mem, ids, ctxs


def _passes(model, mem, ids, ctxs):
    return {"ar": model.ar(mem, ids), "nar": model.nar(mem, L), "refine": model.refine(mem, ctxs)}


@functools.lru_cache(maxsize=None)
def _ref(key):
    cfg, sd, mem, ids, ctxs = _case(key)
    return _passes(MapsReference(cfg, sd), mem, ids, ctxs)


@functools.lru_cache(maxsize=None)
def _stats(key, variant):
    cfg, sd, mem, ids, ctxs = _case(key)
    m = MapsReference(cfg, sd, accum=torch.float32) if variant == "fp32" else MapsReference(cfg, sd, bug=variant)
    got = _passes(m, mem, ids, ctxs)
    ref = _ref(key)
    return {k: map_stats(got[k], ref[k]) for k in ref}


def _name(key):
    return f"D{key[0]}-depth{key[1]}"


@pytest.mark.parametrize("key", CASES, ids=[_name(k) for k in CASES])
def test_fp64_maps_are_distributions(key):
    for name, m in _ref(key).items():
        assert m.shape == (B, L, 128), name
        assert bool((m >= 0).all())
        assert torch.allclose(m.sum(-1), torch.ones((B, L), dtype=m.dtype), rtol=0, atol=1e-12), name


@pytest.mark.parametrize("key", CASES, ids=[_name(k) for k in CASES])
def test_fp32_stand_in_is_inside_every_bound_by_2x(key):
    for name, s in _stats(key, "fp32").items():
        print(format_stats(f"{_name(key)} fp32 stand-in {name}", s))
        assert max(excess(s).values()) <= 0.5, (name, excess(s), BOUNDS)


BUG_CASES = [(key, bug) for key in CASES for bug in sorted(BUGS) if bug != "layer0" or key[1] > 1]


@pytest.mark.parametrize("key,bug", BUG_CASES, ids=[f"{_name(k)}-{b}" for k, b in BUG_CASES])
def test_every_bug_exceeds_a_bound_by_2x(key, bug):
    stats = _stats(key, bug)
    for name in BUG_SCHEDULES[bug]:
        print(format_stats(f"{_name(key)} {bug} {name}", stats[name]))
    for bounds in (BOUNDS, GOLDEN_BOUNDS):
        worst = min(max(excess(stats[name], bounds).values()) for name in BUG_SCHEDULES[bug])
        assert worst >= 2.0, (BUGS[bug], bounds, {k: excess(s, bounds) for k, s in stats.items()})
