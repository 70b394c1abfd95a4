"""Generates tests/golden/beam/*.pt: the beams of tests/beam_oracle.py in fp64, driven by the reference's own modules
(strhub.models.parseq.model.PARSeq and strhub.models.vitstr.model.ViTSTR under oracle/timm_shim.py).  Run where the
reference tree exists:

    python tests/make_golden_beam.py

PARSeq: the logits of a slot at step i are those of the reference's AR step (model.py:124-142) for its own prefix:
model.decode([BOS, prefix], memory, tgt_mask[:i+1, :i+1], tgt_query=pos_queries[:, i:i+1],
tgt_query_mask=query_mask[i:i+1, :i+1]) then model.head.  ViTSTR: the image's position-i row of head(norm(x))[:, 1:]
(vitstr/system.py:65-71).

The weights are the seeded synthetic ones of parseq_b200.weights with a seeded head bias (golden_state_dict): with the
reference's random init every logits row is nearly flat (the K-th and (K + 1)-th readings lie 1e-3..1e-1 apart), so no
ranking would be decidable within the engine's error bound; a head bias of sigma 3 with EOS at the top spreads the
classes as a trained head does and ends most readings within a few characters, and since the bias is added in fp32 after
the GEMM it adds no error.  Each golden holds, per image, the hypotheses (character ids, fp64 score), the margin at each
step between the K-th and the (K + 1)-th best entry of the full pool (every allowed child of every active slot and the
finished readings) with the numbers of terms in those two scores, and the
gaps between adjacent final ranks, so that a test can skip what fp32 rounding could reorder; plus what regenerates the
weights, images and allowlists (parseq_b200.weights; `sd_digest` checks them).
"""
from __future__ import annotations

import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

import beam_oracle as BO                                                # noqa: E402
from make_golden_long import charset, make_config_long                  # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images, state_dict_digest  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "beam")
GOLDEN_FILE_LIMIT = 300_000

# (case name, experiment, dec_depth, max_label_length, extra characters, weight seed, sharpness, batch, image seed, K,
#  allowlist kind: None or "mixed")
CASES = [
    ("bm_s_k5_b3",       "parseq",      1, 25, 0,    240, 2.0, 3, 250, 5, None),
    ("bm_ti_c3001_b2",   "parseq-tiny", 1, 25, 2906, 241, 2.0, 2, 251, 4, None),
    ("bm_s_l64_b2",      "parseq",      1, 63, 0,    242, 2.0, 2, 252, 3, None),
    ("bm_d2_s_b2",       "parseq",      2, 25, 0,    243, 2.0, 2, 253, 4, None),
    ("bm_s_sharp_k8_b3", "parseq",      1, 25, 0,    244, 4.0, 3, 254, 8, None),
    ("bm_s_allow_b4",    "parseq",      1, 25, 0,    245, 2.0, 4, 255, 5, "mixed"),
    ("bm_vitstr_s_b3",   "vitstr",      1, 25, 0,    246, 2.0, 3, 256, 6, None),
]


HEAD_BIAS_SIGMA = 8.0


def golden_state_dict(cfg, seed, sharp):
    """init_state_dict(cfg, seed, sharp) with head.bias = N(0, HEAD_BIAS_SIGMA) (seeded), EOS raised to the top + 2."""
    sd = init_state_dict(cfg, seed, sharp=sharp)
    g = torch.Generator().manual_seed(7919 + seed)
    bias = torch.randn(cfg.num_classes, generator=g, dtype=torch.float64) * HEAD_BIAS_SIGMA
    bias[0] = bias[1:].max() + 2.0
    sd["head.bias"] = bias.to(torch.float32)
    return sd


def allowlist_of(case):
    """Mixed per-image allowlists: digits, none, a few letters, the empty string."""
    B = case[7]
    if case[10] is None:
        return None
    base = ["0123456789", None, "abcdeHIJ", ""]
    return [base[b % len(base)] for b in range(B)]


def allowed_of(tok, allow, C):
    if allow is None:
        return None
    ok = [False] * C
    ok[0] = True
    for ch in allow:
        ok[tok._stoi[ch]] = True
    return ok


def distinct_terms(ta, tb):
    """Numbers of terms of target sequences ta, tb (characters, then EOS if the reading ended) outside their common
    prefix."""
    s = 0
    while s < min(len(ta), len(tb)) and ta[s] == tb[s]:
        s += 1
    return len(ta) - s, len(tb) - s


def search(logits_fn, K, num_steps, allowed):
    """beam_oracle.beam_search plus, at each step, the margin between the K-th and (K + 1)-th best entries of the full
    pool and the numbers of log-softmax terms of those two scores that the two do not share (distinct_terms): terms at
    the positions of a common target prefix are the same numbers in both (the engine carries one parent score to all
    its children), so only the others can move the margin."""
    if allowed is not None:
        allowed = [True] + list(allowed[1:])
    slots = [([], 0.0, False)]
    margins, terms = [], []
    for i in range(num_steps):
        active = [s for s in slots if not s[2]]
        if not active:
            break
        rows = logits_fn([s[0] for s in active])
        full = [(s[1], s[0] + [BO.EOS]) for s in slots if s[2]]
        ai = 0
        for prefix, score, done in slots:
            if done:
                continue
            row = [float(v) for v in rows[ai]]
            ai += 1
            lse = BO._lse([row[c] for c in range(len(row)) if allowed is None or allowed[c]])
            full += [(score + (row[c] - lse), prefix + [c]) for c in BO.row_order(row, allowed)]
        full = sorted((v for v in full if not math.isnan(v[0]) and v[0] != BO.NEG_INF), key=lambda v: -v[0])
        if len(full) > K:
            margins.append(full[K - 1][0] - full[K][0])
            terms.append(list(distinct_terms(full[K - 1][1], full[K][1])))
        else:
            margins.append(math.inf)
            terms.append([0, 0])
    hyps = BO.beam_search(logits_fn, K, num_steps, allowed)
    return hyps, margins, terms


def parseq_fn(ref, tok, memory_b, L):
    mask = torch.triu(torch.ones((L, L), dtype=torch.bool), 1)

    def fn(prefixes):
        i = len(prefixes[0])
        assert all(len(p) == i for p in prefixes)
        P = len(prefixes)
        tgt_in = torch.tensor([[tok.bos_id] + list(p) for p in prefixes], dtype=torch.long)
        out = ref.decode(tgt_in, memory_b.expand(P, -1, -1), mask[:i + 1, :i + 1],
                         tgt_query=ref.pos_queries[:, i:i + 1].expand(P, -1, -1), tgt_query_mask=mask[i:i + 1, :i + 1])
        return ref.head(out)[:, 0].tolist()
    return fn


def make(case):
    from oracle import reference_loader as RL
    from parseq_b200.tokenizer import Tokenizer
    name, exp, depth, mll, n_extra, wseed, sharp, B, iseed, K, _ = case
    extra = {} if exp == "vitstr" else {"dec_depth": depth}
    cfg = make_config_long(exp, mll, n_extra, **extra)
    sd = golden_state_dict(cfg, wseed, sharp)
    x = synth_images(cfg, B, iseed).double()
    L = mll + 1
    C = cfg.num_classes
    tok = Tokenizer(cfg.charset_train)
    allow = allowlist_of(case)
    images = []
    with torch.inference_mode():
        if exp == "vitstr":
            ref = RL.build_reference_vitstr(cfg, sd).double()
            logits = ref(x, L + 1)[:, 1:]                          # vitstr/system.py:67-70 at max_length = L - 1
            fns = [(lambda b: (lambda prefixes: [logits[b, len(p)].tolist() for p in prefixes]))(b) for b in range(B)]
        else:
            ref, _ = RL.build_reference_model(cfg, sd)
            ref = ref.double()
            memory = ref.encode(x)
            fns = [parseq_fn(ref, tok, memory[b:b + 1], L) for b in range(B)]
        for b in range(B):
            allowed = allowed_of(tok, None if allow is None else allow[b], C)
            hyps, margins, terms = search(fns[b], K, L, allowed)
            scores = [s for _, s in hyps]
            images.append(dict(ids=[list(p) for p, _ in hyps], scores=torch.tensor(scores, dtype=torch.float64),
                               prune_margins=torch.tensor(margins, dtype=torch.float64),
                               prune_terms=torch.tensor(terms, dtype=torch.int32).reshape(-1, 2),
                               rank_gaps=torch.tensor([scores[k] - scores[k + 1] for k in range(len(scores) - 1)],
                                                      dtype=torch.float64)))
    blob = dict(name=name, experiment=exp, dec_depth=depth, max_label_length=mll, n_extra=n_extra, weight_seed=wseed,
                sharp=sharp, batch=B, image_seed=iseed, beam_width=K, allowlist=allow, sd_digest=state_dict_digest(sd),
                images=images,
                source="reference %s (timm shim), fp64 beams of tests/beam_oracle.py, torch %s CPU"
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
