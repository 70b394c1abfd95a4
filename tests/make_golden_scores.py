"""Generates tests/golden/score/*.pt: candidate-label log-likelihoods computed by the reference's own modules
(strhub.models.parseq.model.PARSeq and strhub.models.vitstr.model.ViTSTR under oracle/timm_shim.py) in fp64.  Run where
the reference tree exists:

    python tests/make_golden_scores.py

PARSeq: for each (image, candidate c = c_1..c_n) the teacher-forced pass of the canonical left-to-right permutation,
as training_step runs it (strhub/models/parseq/system.py:169-197): tgt_in = [BOS, c_1..c_n], the content and query masks
of generate_attn_masks (system.py:153-167) for perm = [0, 1, .., n + 1], model.encode / model.decode / model.head, then
log_softmax and the gather of the targets t = (c_1..c_n, EOS).  ViTSTR: log_softmax of head(norm(x))[:, 1:]
(vitstr/system.py:65-71) gathered at t.  Each golden holds the fp64 scores [M] and per-position terms [M, L] (0 past n),
the candidates per image, and what regenerates weights and images (parseq_b200.weights; `sd_digest` checks them).
"""
from __future__ import annotations

import os
import random
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

from make_golden_long import charset, make_config_long                 # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images, state_dict_digest  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "score")
GOLDEN_FILE_LIMIT = 300_000


def words(cs: str, seed: int, k: int, lo: int, hi: int):
    r = random.Random(seed)
    return ["".join(r.choice(cs) for _ in range(r.randint(lo, hi))) for _ in range(k)]


def ragged(cs: str, seed: int, B: int, mll: int):
    """Per image: the empty label, one character, a label of max_label_length characters and a few seeded words."""
    r = random.Random(seed)
    out = []
    for b in range(B):
        extra = words(cs, seed * 100 + b, r.randint(1, 5), 2, 12)
        out.append(["", r.choice(cs), "".join(r.choice(cs) for _ in range(mll))] + extra)
    return out


# (case name, experiment, dec_depth, max_label_length, extra characters, weight seed, sharpness, batch, image seed,
#  candidates: "ragged" (per image) or "lexicon" (one list shared by every image))
CASES = [
    ("sc_s_ragged_b4",   "parseq",      1, 25, 0,    140, 0.0, 4, 150, "ragged"),
    ("sc_ti_lexicon_b3", "parseq-tiny", 1, 25, 0,    141, 0.0, 3, 151, "lexicon"),
    ("sc_ti_c3001_b2",   "parseq-tiny", 1, 25, 2906, 142, 0.0, 2, 152, "ragged"),
    ("sc_s_l64_b2",      "parseq",      1, 63, 0,    143, 0.0, 2, 153, "ragged"),
    ("sc_d2_s_b3",       "parseq",      2, 25, 0,    144, 0.0, 3, 154, "ragged"),
    ("sc_s_sharp_b4",    "parseq",      1, 25, 0,    145, 4.0, 4, 155, "lexicon"),
    ("sc_vitstr_s_b3",   "vitstr",      1, 25, 0,    146, 0.0, 3, 156, "ragged"),
]


def candidates_of(case):
    name, exp, depth, mll, n_extra, wseed, sharp, B, iseed, kind = case
    cs = charset(n_extra)
    if kind == "lexicon":
        lex = words(cs[:94], wseed, 12, 3, 12) + ["", "a"]
        return [list(lex) for _ in range(B)]
    return ragged(cs, wseed, B, mll)


def attn_masks(sz: int):
    """generate_attn_masks (system.py:153-167) for the canonical permutation perm = [0, 1, .., sz - 1]."""
    perm = torch.arange(sz)
    mask = torch.zeros((sz, sz), dtype=torch.bool)
    for i in range(sz):
        mask[perm[i], perm[i + 1:]] = True
    content_mask = mask[:-1, :-1].clone()
    mask[torch.eye(sz, dtype=torch.bool)] = True
    query_mask = mask[1:, :-1]
    return content_mask, query_mask


def parseq_terms(ref, tok, x, cands, L):
    terms = []
    with torch.inference_mode():
        memory = ref.encode(x)
        for b, row in enumerate(cands):
            for c in row:
                n = len(c)
                tgt = tok.encode([c])                       # [BOS, c_1..c_n, EOS]
                tgt_in, tgt_out = tgt[:, :-1], tgt[:, 1:]
                content_mask, query_mask = attn_masks(n + 2)
                out = ref.decode(tgt_in, memory[b:b + 1], content_mask, None, None, query_mask)
                lp = torch.log_softmax(ref.head(out), -1)[0]
                t = torch.zeros(L, dtype=torch.float64)
                t[:n + 1] = lp.gather(1, tgt_out[0][:, None])[:, 0]
                terms.append(t)
    return torch.stack(terms)


def vitstr_terms(ref, tok, x, cands, L):
    terms = []
    with torch.inference_mode():
        lp = torch.log_softmax(ref(x, L + 1)[:, 1:], -1)      # vitstr/system.py:67-70 at max_length = L - 1
        for b, row in enumerate(cands):
            for c in row:
                n = len(c)
                ids = torch.tensor(tok._tok2ids(c) + [0], dtype=torch.long)
                t = torch.zeros(L, dtype=torch.float64)
                t[:n + 1] = lp[b, :n + 1].gather(1, ids[:, None])[:, 0]
                terms.append(t)
    return torch.stack(terms)


def make(case):
    from oracle import reference_loader as RL
    name, exp, depth, mll, n_extra, wseed, sharp, B, iseed, kind = case
    extra = {} if exp == "vitstr" else {"dec_depth": depth}
    cfg = make_config_long(exp, mll, n_extra, **extra)
    sd = init_state_dict(cfg, wseed, sharp=sharp)
    x = synth_images(cfg, B, iseed).double()
    cands = candidates_of(case)
    L = mll + 1
    if exp == "vitstr":
        from parseq_b200.tokenizer import Tokenizer
        ref = RL.build_reference_vitstr(cfg, sd).double()
        terms = vitstr_terms(ref, Tokenizer(cfg.charset_train), x, cands, L)
    else:
        ref, tok = RL.build_reference_model(cfg, sd)
        terms = parseq_terms(ref.double(), tok, x, cands, L)
    scores = terms.sum(-1)
    blob = dict(name=name, experiment=exp, dec_depth=depth, max_label_length=mll, n_extra=n_extra, weight_seed=wseed,
                sharp=sharp, batch=B, image_seed=iseed, sd_digest=state_dict_digest(sd), candidates=cands,
                scores=scores, terms=terms,
                source="reference %s (timm shim), fp64 teacher-forced scores, torch %s CPU"
                       % ("strhub.models.vitstr.model.ViTSTR" if exp == "vitstr" else "strhub.models.parseq.model.PARSeq",
                          torch.__version__))
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    print(f"{name:18s} C={cfg.num_classes} M={len(scores)} scores [{scores.min().item():.2f}, {scores.max().item():.2f}] "
          f"{size / 1e3:.0f} KB")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        make(case)
