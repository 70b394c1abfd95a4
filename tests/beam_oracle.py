"""fp64 reference of the engine's beam search rule (include/parseq_b200.h, parseq_beam_search).

`beam_search(logits_fn, K, num_steps, ...)` runs one search per image over a callable that returns the next-token
logits of a batch of prefixes: logits_fn(prefixes) -> [len(prefixes), C], prefixes being lists of character ids (BOS
not included).  The rule:
  - K slots; slot 0 starts as the empty prefix with score 0, the others empty.
  - Step i: each active slot's row gives LSE = logsumexp over the allowed classes (NaN if one is NaN or +inf, as in
    score()), terms logit - LSE, children parent + term; the slot expands its K best classes in row order (NaN logits
    first, then logit descending, ties to the lower class); masked classes and -inf logits never expand.
  - EOS (class 0) finishes a child with its length; a child with num_steps characters is finished too.
  - The pool, in slot order (a finished slot itself, an active slot its expansions), keeps its K best by a stable sort on
    the score; NaN ranks after every number, -inf is never kept.
"""
from __future__ import annotations

import itertools
import math
from typing import Callable, List, Optional, Sequence, Tuple

EOS = 0
NEG_INF = float("-inf")


def _lse(vals: Sequence[float]) -> float:
    if any(math.isnan(v) or v == float("inf") for v in vals):
        return float("nan")
    m = max(vals, default=NEG_INF)
    if m == NEG_INF:
        return NEG_INF
    return m + math.log(sum(math.exp(v - m) for v in vals))


def row_order(row: Sequence[float], allowed: Optional[Sequence[bool]] = None) -> List[int]:
    """The classes a row expands, in expansion order (masked and -inf classes left out)."""
    cls = [c for c in range(len(row)) if (allowed is None or allowed[c]) and row[c] != NEG_INF]
    nan = [c for c in cls if math.isnan(row[c])]
    num = sorted((c for c in cls if not math.isnan(row[c])), key=lambda c: (-row[c], c))
    return nan + num


def rank_key(score: float):
    return (1, 0.0) if math.isnan(score) else (0, -score)


def beam_search(logits_fn: Callable[[List[List[int]]], Sequence[Sequence[float]]], K: int, num_steps: int,
                allowed: Optional[Sequence[bool]] = None) -> List[Tuple[List[int], float]]:
    """Hypotheses (character ids without EOS, score) of one image, best first (at most K)."""
    if allowed is not None:
        allowed = [True] + list(allowed[1:])          # EOS is always allowed
    # slot: (prefix, score, finished)
    slots: List[Tuple[List[int], float, bool]] = [([], 0.0, False)]
    for i in range(num_steps):
        active = [s for s in slots if not s[2]]
        if not active:
            break
        rows = logits_fn([s[0] for s in active])
        pool = []
        ai = 0
        for prefix, score, done in slots:
            if done:
                pool.append((prefix, score, True))
                continue
            row = [float(v) for v in rows[ai]]
            ai += 1
            lse = _lse([row[c] for c in range(len(row)) if allowed is None or allowed[c]])
            for c in row_order(row, allowed)[:K]:
                child = score + (row[c] - lse)
                if c == EOS:
                    pool.append((prefix, child, True))
                else:
                    pool.append((prefix + [c], child, i + 1 == num_steps))
        pool = [p for p in pool if p[1] != NEG_INF]
        slots = sorted(pool, key=lambda p: rank_key(p[1]))[:K]        # sorted() is stable
    return [(p, s) for p, s, _ in slots]


def sequence_logprob(logits_fn, seq: Sequence[int], num_steps: int, allowed: Optional[Sequence[bool]] = None) -> float:
    """Teacher-forced log-likelihood of c_1..c_n (then EOS unless n == num_steps) under the same LSE rule."""
    if allowed is not None:
        allowed = [True] + list(allowed[1:])
    total = 0.0
    targets = list(seq) + ([EOS] if len(seq) < num_steps else [])
    for i, t in enumerate(targets):
        row = [float(v) for v in logits_fn([list(seq[:i])])[0]]
        lse = _lse([row[c] for c in range(len(row)) if allowed is None or allowed[c]])
        total += row[t] - lse
    return total


def exhaustive(logits_fn, num_classes: int, num_steps: int, allowed: Optional[Sequence[bool]] = None):
    """Every finite reading (ids without EOS) with its log-likelihood, best first (ties: the order beam search builds)."""
    chars = [c for c in range(1, num_classes) if allowed is None or allowed[c]]
    out = []
    for n in range(num_steps + 1):
        for seq in itertools.product(chars, repeat=n):
            out.append((list(seq), sequence_logprob(logits_fn, seq, num_steps, allowed)))
    return sorted(out, key=lambda p: -p[1])
