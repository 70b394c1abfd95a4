"""The rule of the orientation search (parseq_forward_crops_oriented, include/parseq_b200.h) restated in fp64, and the
confidence it ranks readings by: the reference's sequence confidence (strhub/models/base.py:132-142 `_eval_step`:
logits.softmax(-1) -> Tokenizer.decode -> probs.prod(), the EOS probability included).

Rule.  Orientations o_0 .. o_{R-1}; every crop is read at o_0 and keeps that reading when its confidence is >= t
(min_confidence).  Otherwise (always, without t) it also reads o_1 .. o_{R-1} and takes the reading of highest
confidence; ties go to the earlier orientation, NaN ranks below every number."""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import numpy as np


def better(c: float, best: float) -> bool:
    """Does confidence c beat the best so far?  Strictly greater, or a number against NaN."""
    c, best = float(c), float(best)
    if math.isnan(c):
        return False
    return math.isnan(best) or c > best


def rereads(c0: float, min_confidence: Optional[float]) -> bool:
    """Is a crop whose first reading has confidence c0 read in the other orientations?"""
    return min_confidence is None or not (float(c0) >= float(min_confidence))


def choose(confidences: Sequence[float], min_confidence: Optional[float] = None) -> int:
    """Index of the chosen orientation for one crop, given the confidence of its reading in each orientation."""
    if not rereads(confidences[0], min_confidence):
        return 0
    best, k = confidences[0], 0
    for r in range(1, len(confidences)):
        if better(confidences[r], best):
            best, k = confidences[r], r
    return k


def select(confidences: np.ndarray, min_confidence: Optional[float] = None) -> Tuple[np.ndarray, np.ndarray]:
    """confidences [N, R] -> (chosen orientation index [N], re-read mask [N])."""
    conf = np.asarray(confidences, dtype=np.float64)
    pick = np.array([choose(row, min_confidence) for row in conf], dtype=np.int64)
    rr = np.array([rereads(row[0], min_confidence) for row in conf], dtype=bool)
    return pick, rr


def reference_confidence(logits: np.ndarray, eos_id: int = 0) -> Tuple[float, int]:
    """fp64 replay of `_eval_step`'s confidence of one image: logits [L, C] -> (product of the max softmax probability
    of each position up to and including the first EOS, length = index of that EOS or L).  A row whose maximum is not
    finite has an all-NaN softmax in torch: id 0 with probability NaN."""
    x = np.asarray(logits, dtype=np.float64)
    conf, L = 1.0, x.shape[0]
    for i in range(L):
        row = x[i]
        m = np.max(row) if not np.isnan(row).any() else np.nan
        if not np.isfinite(m):
            conf *= math.nan
            i_d = 0
        else:
            p = np.exp(row - m)
            conf *= 1.0 / p.sum()
            i_d = int(np.argmax(row))
        if i_d == eos_id:
            return conf, i
    return conf, L
