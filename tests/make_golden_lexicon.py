"""Generates tests/golden/lexicon/*.pt: lexicon-constrained beams of tests/lexicon_oracle.py in fp64, driven by the
reference's own modules exactly as tests/make_golden_beam.py drives them (same logits functions, the same seeded head
bias).  Run where the reference tree exists:

    python tests/make_golden_lexicon.py

Each golden holds its lexicon (one word list for every image, or one per image), and per image the hypotheses
(character ids, fp64 score), the margin at each step between the K-th and the (K + 1)-th best entry of the full pool
(every expandable child of every active slot and the finished readings) with the numbers of terms in those two scores
that the two do not share, so that a test can skip what fp32 rounding could reorder.
"""
from __future__ import annotations

import math
import os
import random
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

import lexicon_oracle as LO                                             # noqa: E402
from make_golden_beam import GOLDEN_FILE_LIMIT, allowed_of, distinct_terms, golden_state_dict, parseq_fn  # noqa: E402
from make_golden_long import charset, make_config_long                  # noqa: E402
from parseq_b200.weights import synth_images, state_dict_digest         # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "lexicon")

# (case name, experiment, dec_depth, max_label_length, extra characters, weight seed, sharpness, batch, image seed, K,
#  lexicon kind: "shared" (300 words) / "per-image" (50 words each) / "long" (200 words of 20..60 characters),
#  allowlist kind: None or "mixed")
CASES = [
    ("lx_s_shared_b3",    "parseq",      1, 25, 0,    260, 2.0, 3, 270, 5, "shared",    None),
    ("lx_s_per_b3",       "parseq",      1, 25, 0,    261, 2.0, 3, 271, 4, "per-image", None),
    ("lx_s_allow_b4",     "parseq",      1, 25, 0,    262, 2.0, 4, 272, 5, "shared",    "mixed"),
    ("lx_d2_s_b2",        "parseq",      2, 25, 0,    263, 2.0, 2, 273, 4, "shared",    None),
    ("lx_s_l64_b2",       "parseq",      1, 63, 0,    264, 2.0, 2, 274, 3, "long",      None),
    ("lx_ti_c3001_b2",    "parseq-tiny", 1, 25, 2906, 265, 2.0, 2, 275, 4, "shared",    None),
    ("lx_vitstr_s_b3",    "vitstr",      1, 25, 0,    266, 2.0, 3, 276, 6, "shared",    None),
]


def lexicon_of(case, cs):
    """The case's lexicon: seeded words over charset cs (one list, or one per image), with "" and prefix chains."""
    kind, B, seed = case[10], case[7], case[5]
    rng = random.Random(9001 + seed)

    def words(n, lo, hi):
        out = {"", cs[:1], cs[:2], cs[:3]}
        while len(out) < n:
            out.add("".join(rng.choice(cs) for _ in range(rng.randint(lo, hi))))
        return sorted(out)
    if kind == "per-image":
        return [words(50, 1, 8) for _ in range(B)]
    if kind == "long":
        return words(200, 20, 60)
    return words(300, 1, 8)


def allowlist_of(case):
    if case[11] is None:
        return None
    base = ["0123456789", None, "abcdeHIJ", ""]
    return [base[b % len(base)] for b in range(case[7])]


def margins_of(pools, K):
    """Per step, the margin between the K-th and (K + 1)-th best entries of the full pool (lexicon_oracle's `pools`)
    and the numbers of terms of those two scores that the two do not share (as make_golden_beam.search)."""
    margins, terms = [], []
    for full in pools:
        if len(full) > K:
            margins.append(full[K - 1][0] - full[K][0])
            terms.append(list(distinct_terms(full[K - 1][1], full[K][1])))
        else:
            margins.append(math.inf)
            terms.append([0, 0])
    return margins, terms


def make(case):
    from oracle import reference_loader as RL
    from parseq_b200.lexicon import build_trie
    from parseq_b200.tokenizer import Tokenizer
    name, exp, depth, mll, n_extra, wseed, sharp, B, iseed, K, _, _ = case
    extra = {} if exp == "vitstr" else {"dec_depth": depth}
    cfg = make_config_long(exp, mll, n_extra, **extra)
    sd = golden_state_dict(cfg, wseed, sharp)
    x = synth_images(cfg, B, iseed).double()
    L = mll + 1
    C = cfg.num_classes
    tok = Tokenizer(cfg.charset_train)
    cs = charset(n_extra)
    lexicon = lexicon_of(case, cs)
    rows = lexicon if isinstance(lexicon[0], list) else [lexicon] * B
    allow = allowlist_of(case)
    images = []
    with torch.inference_mode():
        if exp == "vitstr":
            ref = RL.build_reference_vitstr(cfg, sd).double()
            logits = ref(x, L + 1)[:, 1:]
            fns = [(lambda b: (lambda prefixes: [logits[b, len(p)].tolist() for p in prefixes]))(b) for b in range(B)]
        else:
            ref, _ = RL.build_reference_model(cfg, sd)
            ref = ref.double()
            memory = ref.encode(x)
            fns = [parseq_fn(ref, tok, memory[b:b + 1], L) for b in range(B)]
        for b in range(B):
            allowed = allowed_of(tok, None if allow is None else allow[b], C)
            trie = build_trie([[tok._tok2ids(w) for w in rows[b]]])
            pools = []
            hyps = LO.lexicon_beam_search(fns[b], K, L, *trie, root=0, allowed=allowed, pools=pools)
            margins, terms = margins_of(pools, K)
            images.append(dict(ids=[list(p) for p, _ in hyps],
                               scores=torch.tensor([s for _, s in hyps], dtype=torch.float64),
                               prune_margins=torch.tensor(margins, dtype=torch.float64),
                               prune_terms=torch.tensor(terms, dtype=torch.int32).reshape(-1, 2)))
    blob = dict(name=name, experiment=exp, dec_depth=depth, max_label_length=mll, n_extra=n_extra, weight_seed=wseed,
                sharp=sharp, batch=B, image_seed=iseed, beam_width=K, lexicon=lexicon, allowlist=allow,
                sd_digest=state_dict_digest(sd), images=images,
                source="reference %s (timm shim), fp64 lexicon beams of tests/lexicon_oracle.py, torch %s CPU"
                       % ("strhub.models.vitstr.model.ViTSTR" if exp == "vitstr" else "strhub.models.parseq.model.PARSeq",
                          torch.__version__))
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    print(f"{name:18s} C={C} K={K} hyps={[len(im['ids']) for im in images]} "
          f"min margin {min(float(im['prune_margins'].min()) for im in images):.3g} {size / 1e3:.0f} KB", flush=True)


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    only = sys.argv[1:]
    for case in CASES:
        if not only or case[0] in only:
            make(case)
