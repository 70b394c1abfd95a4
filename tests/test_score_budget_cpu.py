"""Where the error budget of candidate scores comes from (no GPU): tests/score_budget.py derives per-term bounds from the
decoder's logit bounds (decoder_reference.BOUNDS).  Here, on the scoring pass (teacher-forced, causal, one row per
candidate position) with sharp (x4) attention weights and a memory from the oracle's encoder, the fp32 stand-in stays
within half of every term bound, and each of the self_mask_leak and pos_query_shift bugs exceeds one by 2x or more."""
import functools

import pytest
import torch

from decoder_reference import DecoderReference, DepthDecoderReference
from score_budget import SCORE_BUGS, TERM_BOUNDS, forcing, model_terms, term_excess, term_stats, words

EXPERIMENT = {192: "parseq-tiny", 384: "parseq", 768: "parseq-base-48x160"}
M = 8
CASES = [(192, 1), (384, 1), (384, 2)]


@functools.lru_cache(maxsize=None)
def _case(key):
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.config import make_config
    from parseq_b200.tokenizer import Tokenizer
    from parseq_b200.weights import init_state_dict, synth_images
    D, depth = key
    cfg = make_config(EXPERIMENT[D], enc_depth=2, dec_depth=depth)
    sd = init_state_dict(cfg, 3, sharp=4.0)
    enc = make_config(EXPERIMENT[D], enc_depth=2)
    mem = ParseqOracle(enc, init_state_dict(enc, 3, sharp=4.0), "fp32").encode(synth_images(cfg, M, 7))
    mem = mem.to(torch.bfloat16).float()
    tok = Tokenizer(cfg.charset_train)
    ids, tgt, valid = forcing(tok, words(cfg.charset_train, 5, M, cfg.max_label_length), cfg.max_label_length + 1)
    model = DepthDecoderReference if depth > 1 else DecoderReference
    ref_logits = model(cfg, sd).ar(mem, ids)
    return model, cfg, sd, mem, ids, tgt, valid, ref_logits, model_terms(ref_logits, tgt, valid)


@pytest.mark.parametrize("key", CASES, ids=lambda k: f"D{k[0]}-depth{k[1]}")
def test_fp32_stand_in_within_half_of_the_term_bounds(key):
    model, cfg, sd, mem, ids, tgt, valid, ref_logits, ref = _case(key)
    got = model_terms(model(cfg, sd, accum=torch.float32).ar(mem, ids), tgt, valid)
    s = term_stats(got, ref, ref_logits, valid)
    print(key, s)
    assert max(term_excess(s, key).values()) <= 0.5, (s, TERM_BOUNDS[key])


@pytest.mark.parametrize("bug", SCORE_BUGS)
@pytest.mark.parametrize("key", CASES, ids=lambda k: f"D{k[0]}-depth{k[1]}")
def test_scoring_bugs_exceed_the_term_bounds(key, bug):
    model, cfg, sd, mem, ids, tgt, valid, ref_logits, ref = _case(key)
    got = model_terms(model(cfg, sd, bug=bug).ar(mem, ids), tgt, valid)
    s = term_stats(got, ref, ref_logits, valid)
    print(key, bug, s)
    assert max(term_excess(s, key).values()) >= 2.0, (bug, s, TERM_BOUNDS[key])
