"""The error budget of candidate scores against the fp64 decoder model of tests/decoder_reference.py.  TEST HELPER.

A score's term at position i is log_softmax(logits_i)[t_i] = logit_i[t_i] - logsumexp(logits_i).  To first order the
error of logsumexp is the softmax-weighted mean of the row's logit errors, so

    |d term| <= |d logit[t]| + sum_c p_c |d logit_c|.

The first summand is one draw from the logit errors that decoder_reference.BOUNDS bounds (relative to sigma, the standard
deviation of the model's logits); the second is a weighted average of such draws, typically of the size of their mean,
at most the row's largest.  Hence the term bounds: median <= median + mean of the logit bounds, mean <= 2 x mean,
p99 <= 2 x p99.  tests/test_score_budget_cpu.py shows the fp32 stand-in (a correct decoder's noise) within half of them
and the injected self_mask_leak and pos_query_shift bugs above them by 2x or more; tests/test_gpu_score.py holds the
engine's scores to them.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch

from decoder_reference import BOUNDS

TERM_BOUNDS: Dict[Tuple[int, int], Dict[str, float]] = {
    k: {"p50": b["p50"] + b["mean"], "mean": 2 * b["mean"], "p99": 2 * b["p99"]} for k, b in BOUNDS.items()}
SCORE_BUGS = ("self_mask_leak", "pos_query_shift")


def words(cs: str, seed: int, k: int, max_len: int) -> List[str]:
    """k seeded words whose lengths spread over 0..max_len."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for j in range(k):
        n = (j * 7 + int(torch.randint(0, 3, (), generator=g))) % (max_len + 1)
        out.append("".join(cs[int(i)] for i in torch.randint(0, len(cs), (n,), generator=g)))
    return out


def forcing(tok, cands: List[str], L: int):
    """(context ids [M, L] = BOS, c_1..c_n, PAD..., targets [M, L] = c_1..c_n, EOS, 0..., valid [M, L] = i <= n)."""
    M = len(cands)
    ids = torch.full((M, L), tok.pad_id, dtype=torch.long)
    tgt = torch.zeros((M, L), dtype=torch.long)
    valid = torch.zeros((M, L), dtype=torch.bool)
    for m, c in enumerate(cands):
        ch = tok._tok2ids(c)
        ids[m, 0] = tok.bos_id
        ids[m, 1:1 + len(ch)] = torch.tensor(ch, dtype=torch.long)
        tgt[m, :len(ch) + 1] = torch.tensor(ch + [tok.eos_id], dtype=torch.long)
        valid[m, :len(ch) + 1] = True
    return ids, tgt, valid


def model_terms(logits: torch.Tensor, tgt: torch.Tensor, valid: torch.Tensor) -> torch.Tensor:
    """The terms [M, L] of logits [M, L, C] (0 where not valid)."""
    lp = torch.log_softmax(logits.double(), -1).gather(2, tgt.to(logits.device)[..., None])[..., 0]
    return torch.where(valid.to(lp.device), lp, torch.zeros_like(lp))


def term_stats(got: torch.Tensor, ref: torch.Tensor, ref_logits: torch.Tensor, valid: torch.Tensor) -> Dict[str, float]:
    """sigma of the model's logits over the scored rows, and the median, mean, p99 and max of |got - ref| over the scored
    terms relative to it."""
    v = valid.to(ref.device)
    sigma = ref_logits.double()[v].std().item()
    d = (got.to(ref.device, torch.float64) - ref.double()).abs()[v]
    n = d.numel()
    return {"sigma": sigma, "p50": d.kthvalue((n + 1) // 2).values.item() / sigma, "mean": d.mean().item() / sigma,
            "p99": d.kthvalue(max(1, math.ceil(0.99 * n))).values.item() / sigma, "max": d.max().item() / sigma}


def term_excess(stats: Dict[str, float], key: Tuple[int, int]) -> Dict[str, float]:
    return {k: stats[k] / b for k, b in TERM_BOUNDS[key].items()}
