"""Where the decoder's error budget comes from (no GPU).

For each decoder width (and PARSeq-S at depth 2), with sharp (x4) attention weights and a memory from the oracle's
encoder (depth 2), the fp64 rounding-point model of tests/decoder_reference.py runs teacher-forced AR and one refinement
pass over random ids.  Two kinds of variant are compared with it, pass by pass, on decoder_reference.budget_stats:
  * the fp32 stand-in (same rounding points and engine functions, fp32 arithmetic), i.e. what a correct decoder looks
    like: it must stay within half of every bound of decoder_reference.BOUNDS;
  * each injected bug of decoder_reference.BUGS: it must exceed some bound by 2x or more in some pass.
So the bounds that tests/test_gpu_decoder_isolated.py holds the engine to sit at least 2x above the stand-in's noise and
at least 2x below each of these mistakes, except where EXCLUDED says, with the numbers, that no bound can be: at
D >= 384 and at depth 2 the three smallest bugs (ln_eps, cross_extra_zero_key, cross_q_bf16) and self_q_bf16, and at
depth 2 also norm_qc_eps, where a correct decoder's noise is within 2x of them.  At D = 192 they exceed the bounds by
2x or more while the engine stays 1.8x or more below them.  The probes of tests/probe_models.py cover every excluded
entry (tests/test_probe_separation_cpu.py)."""
import functools

import pytest
import torch

from decoder_reference import (BOUNDS, BUGS, DecoderReference, DepthDecoderReference, budget_stats, excess,
                               forced_ar_ids, format_stats, refine_context)

EXPERIMENT = {192: "parseq-tiny", 384: "parseq", 768: "parseq-base-48x160"}
B, L = 8, 26

# (embed_dim, dec_depth) -> bugs that no bound separates from a correct decoder there.  Medians |d| / sigma of the AR
# pass: the bug, the fp32 stand-in, and the engine's largest over the GPU test's cases, which sets the bound's floor.
_SMALL = ("ln_eps", "cross_extra_zero_key", "cross_q_bf16")
EXCLUDED = {
    # bugs 2.23e-3 / 2.15e-3 / 2.29e-3; the stand-in's median is 4e-7, but the engine's reaches 1.07e-3 (the 2-class head;
    # 3e-4 to 6e-4 elsewhere), so the median bound is 1.6e-3 and these bugs exceed it by 1.3x to 1.4x only.
    # self_q_bf16: median 3.03e-3, 1.9x the bound
    (384, 1): _SMALL + ("self_q_bf16",),
    # bugs 2.05e-3 / 9.1e-4 / 2.61e-3; stand-in 2.2e-4; the engine reaches 1.9e-3 (chain at L = 64), so the median
    # bound is 2.6e-3 and the bugs' means (2.5e-3 / 1.3e-3 / 3.1e-3) stay under the engine's 2.4e-3 x 1.5 too.
    # self_q_bf16: median 3.86e-3, 1.5x the bound
    (768, 1): _SMALL + ("self_q_bf16",),
    # bugs 3.1e-3 / 3.1e-3 / 3.2e-3; the stand-in's own median is 1.7e-3: a second layer carries the flips of the first
    # into every row, so the bound cannot be below 3.5e-3.  norm_qc_eps: median 5.74e-3, 1.6x the bound;
    # self_q_bf16: median 3.82e-3, 1.1x
    (384, 2): _SMALL + ("norm_qc_eps", "self_q_bf16"),
}
CASES = sorted(BOUNDS)


@functools.lru_cache(maxsize=None)
def _case(key):
    """(model class, config, state_dict, bf16 memory, AR forcing, refine context, fp64 logits of both passes)."""
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.config import make_config
    from parseq_b200.weights import init_state_dict, synth_images
    D, depth = key
    cfg = make_config(EXPERIMENT[D], enc_depth=2, dec_depth=depth)
    sd = init_state_dict(cfg, 3, sharp=4.0)
    enc = make_config(EXPERIMENT[D], enc_depth=2)        # the oracle's encoder restates depth-1 configs
    mem = ParseqOracle(enc, init_state_dict(enc, 3, sharp=4.0), "fp32").encode(synth_images(cfg, B, 7))
    mem = mem.to(torch.bfloat16).float()
    bos, C = cfg.num_tokens - 2, cfg.num_classes
    forced = forced_ar_ids(B, L, C, bos, 1)
    ctx = refine_context(B, L, C, bos, [1, 5, 12, 20, 25, None], 2)
    model = DepthDecoderReference if depth > 1 else DecoderReference
    return model, cfg, sd, mem, forced, ctx, _passes(model(cfg, sd), mem, forced, ctx)


def _passes(model, mem, forced, ctx):
    return {"ar": model.ar(mem, forced), "refine": model.refine(mem, ctx)}


@functools.lru_cache(maxsize=None)
def _stats(key, variant):
    model, cfg, sd, mem, forced, ctx, ref = _case(key)
    m = model(cfg, sd, accum=torch.float32) if variant == "fp32" else model(cfg, sd, bug=variant)
    got = _passes(m, mem, forced, ctx)
    return {k: budget_stats(got[k], ref[k]) for k in ref}


def _name(key):
    return f"D{key[0]}-depth{key[1]}"


@pytest.mark.parametrize("key", CASES, ids=[_name(k) for k in CASES])
def test_fp32_stand_in_is_inside_every_bound_by_2x(key):
    for name, s in _stats(key, "fp32").items():
        print(format_stats(f"{_name(key)} fp32 stand-in {name}", s))
        assert max(excess(s, key).values()) <= 0.5, (name, excess(s, key))


@pytest.mark.parametrize("bug", sorted(BUGS))
@pytest.mark.parametrize("key", CASES, ids=[_name(k) for k in CASES])
def test_every_bug_exceeds_a_bound_by_2x(key, bug):
    """...and the bugs left out at a configuration really are within 2x there, so the list cannot go stale."""
    stats = _stats(key, bug)
    for name, s in stats.items():
        print(format_stats(f"{_name(key)} {bug} {name}", s))
    worst = max(max(excess(s, key).values()) for s in stats.values())
    if bug in EXCLUDED.get(key, ()):
        assert worst < 2.0, (bug, "separates now: take it off EXCLUDED", worst)
    else:
        assert worst >= 2.0, (BUGS[bug], {k: excess(s, key) for k, s in stats.items()})


def test_teacher_forced_ar_loop_is_one_causal_pass():
    """The single causal pass of DecoderReference.ar equals the reference's step-by-step loop (model.py:119-147: step i
    decodes query i over context 0..i), and the depth-N model at depth 1 equals the depth-1 model."""
    model, cfg, sd, mem, forced, ctx, ref = _case((192, 1))
    m = DecoderReference(cfg, sd)
    memr = m._memory(mem)
    ids = forced.long()
    steps = [m._decode(ids[:, : i + 1], memr, m._pos(B, L)[:, i: i + 1], None, None) for i in range(L)]
    assert torch.allclose(torch.cat(steps, dim=1), ref["ar"], rtol=0, atol=1e-10)
    d = DepthDecoderReference(cfg, sd)
    assert torch.allclose(d.ar(mem, forced), ref["ar"], rtol=0, atol=1e-10)
    assert torch.allclose(d.refine(mem, ctx), ref["refine"], rtol=0, atol=1e-10)
    assert torch.allclose(d.nar(mem, L), m.nar(mem, L), rtol=0, atol=1e-10)


def test_engine_gelu_is_the_erf_gelu_to_its_stated_accuracy():
    """decoder_reference.engine_gelu restates ptx.cuh gelu_erf: within 1.3e-6 (absolute) of the exact erf-GELU."""
    from decoder_reference import engine_gelu
    x = torch.linspace(-12.0, 12.0, 200_001, dtype=torch.float64)
    assert (engine_gelu(x) - torch.nn.functional.gelu(x)).abs().max().item() <= 1.3e-6
