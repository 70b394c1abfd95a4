"""Generates tests/golden/alignment/*.pt: the cross-attention maps of given labels (forced alignment, parseq_score_args.
attn_maps) computed by the reference's own modules (strhub.models.parseq.model.PARSeq under oracle/timm_shim.py) in
fp64.  Run where the reference tree exists:

    python tests/make_golden_alignment.py

For each (image, candidate c = c_1..c_n): model.encode, then model.decode of tgt_in = [BOS, c_1..c_n] under the content
and query masks of the canonical left-to-right permutation (generate_attn_masks, strhub/models/parseq/system.py:153-167,
as tests/make_golden_scores.py runs it).  A forward hook on decoder.layers[-1].cross_attn records output[1], the
head-averaged ca_weights of the last layer's query stream (modules.py:74): row i is the map of the query that predicts
t_i (t = c_1..c_n, EOS).  The last layer calls its cross-attention once per decode (its content stream is not updated).
Each golden holds the rows 0..n of every candidate concatenated (fp64 [sum(n + 1), T]), the candidates, and what
regenerates weights and images (`sd_digest` checks them).  The weights are tests/make_golden_attention.py's: seeded
synthetic ones with sharp attention and a seeded head bias.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

from make_golden_attention import golden_state_dict                    # noqa: E402
from make_golden_long import charset, make_config_long                 # noqa: E402
from make_golden_scores import attn_masks, ragged                      # noqa: E402
from parseq_b200.weights import state_dict_digest, synth_images        # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "alignment")
GOLDEN_FILE_LIMIT = 400_000

# (case name, experiment, dec_depth, max_label_length, extra characters, weight seed, sharpness, batch, image seed)
CASES = [
    ("al_s_sharp_b3",    "parseq",             1, 25, 0,    400, 4.0, 3, 410),
    ("al_ti_c3001_b2",   "parseq-tiny",        1, 25, 2906, 401, 4.0, 2, 411),
    ("al_d2_s_b2",       "parseq",             2, 25, 0,    402, 2.0, 2, 412),
    ("al_s_l64_b2",      "parseq",             1, 63, 0,    403, 4.0, 2, 413),
    ("al_p16_b2",        "parseq-patch16-224", 1, 25, 0,    404, 4.0, 2, 414),
]


def config_of(exp, depth, mll, n_extra):
    img = (224, 224) if exp == "parseq-patch16-224" else (32, 128)
    return make_config_long(exp, mll, n_extra, img_size=img, dec_depth=depth)


def candidates_of(case):
    """The first five ragged candidates of tests/make_golden_scores.py per image: the empty label, one character, one of
    max_label_length characters and two seeded words."""
    name, exp, depth, mll, n_extra, wseed, sharp, B, iseed = case
    rows = ragged(charset(n_extra), wseed, B, mll)
    return [r[:5] for r in rows]


def golden_case(name):
    """(blob, cfg, state dict, images, targets, lengths, per_image) of golden `name`: the weights checked by digest, the
    candidates packed as parseq_score takes them (CPU)."""
    from parseq_b200.system import pack_candidates
    from parseq_b200.tokenizer import Tokenizer
    blob = torch.load(os.path.join(OUT, name + ".pt"), weights_only=False)
    cfg = config_of(blob["experiment"], blob["dec_depth"], blob["max_label_length"], blob["n_extra"])
    sd = golden_state_dict(cfg, blob["weight_seed"], blob["sharp"])
    assert state_dict_digest(sd) == blob["sd_digest"]
    x = synth_images(cfg, blob["batch"], blob["image_seed"])
    packed = pack_candidates(Tokenizer(cfg.charset_train), blob["candidates"], blob["batch"], cfg.max_label_length,
                             cfg.num_classes)
    return (blob, cfg, sd, x) + tuple(packed)


def make(case):
    from oracle import reference_loader as RL
    name, exp, depth, mll, n_extra, wseed, sharp, B, iseed = case
    cfg = config_of(exp, depth, mll, n_extra)
    sd = golden_state_dict(cfg, wseed, sharp)
    ref, tok = RL.build_reference_model(cfg, sd)
    ref = ref.double()
    x = synth_images(cfg, B, iseed).double()
    cands = candidates_of(case)
    calls = []
    hook = ref.decoder.layers[-1].cross_attn.register_forward_hook(lambda m, i, o: calls.append(o[1].detach().clone()))
    # grad enabled, as tests/make_golden_attention.py runs it: nn.MultiheadAttention takes its reference path
    memory = ref.encode(x).detach()
    rows = []
    for b, row in enumerate(cands):
        for c in row:
            n = len(c)
            tgt_in = tok.encode([c])[:, :-1]                 # [BOS, c_1..c_n]
            content_mask, query_mask = attn_masks(n + 2)
            calls.clear()
            ref.decode(tgt_in, memory[b:b + 1], content_mask, None, None, query_mask)
            assert len(calls) == 1 and calls[0].shape == (1, n + 1, cfg.num_patches), (name, len(calls))
            rows.append(calls[0][0])
    hook.remove()
    maps = torch.cat(rows).contiguous()
    blob = dict(name=name, experiment=exp, dec_depth=depth, max_label_length=mll, n_extra=n_extra, weight_seed=wseed,
                sharp=sharp, batch=B, image_seed=iseed, sd_digest=state_dict_digest(sd), candidates=cands, maps=maps,
                source="reference strhub.models.parseq.model.PARSeq (timm shim), forward hook on "
                       "decoder.layers[-1].cross_attn, teacher-forced canonical permutation, fp64, torch %s CPU"
                       % torch.__version__)
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    print(f"{name:16s} C={cfg.num_classes} T={cfg.num_patches} rows {maps.shape[0]} {size / 1e3:.0f} KB")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        make(case)
