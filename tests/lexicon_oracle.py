"""fp64 reference of lexicon-constrained beam search (include/parseq_b200.h, parseq_beam_search_lexicon), built on the
rule of tests/beam_oracle.py.

The lexicon is the CSR DAG of parseq_lexicon_desc (first_edge, edge_class, edge_child, terminal) and a root.  Each slot
carries its node v.  Step i: the slot's LSE is beam_oracle's, over the allowed classes of the whole row; its expandable
classes are EOS iff terminal[v], and each edge class c of v iff c is allowed, logit[c] != -inf and i + 1 < num_steps;
it expands its K best expandable classes in row order.  A character moves to the edge's child; EOS finishes the slot.
Pool, stable sort, NaN ranking and -inf handling are beam_oracle's.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import beam_oracle as BO


def lexicon_beam_search(logits_fn, K: int, num_steps: int, first_edge, edge_class, edge_child, terminal, root: int = 0,
                        allowed: Optional[Sequence[bool]] = None, pools: Optional[list] = None) -> List[Tuple[List[int], float]]:
    """Hypotheses (character ids without EOS, score) of one image, best first (at most K).  With a list `pools`, each
    step appends its full pool to it: every finished reading and every expandable child of every active slot (not only
    the K each slot expands), as (score, targets) best first, targets being the characters then EOS if it ended;
    NaN and -inf entries left out.  Its K-th and (K + 1)-th entries give the step's pruning margin."""
    if allowed is not None:
        allowed = [True] + list(allowed[1:])
    edges = {}
    # slot: (prefix, score, finished, node)
    slots = [([], 0.0, False, int(root))]
    for i in range(num_steps):
        active = [s for s in slots if not s[2]]
        if not active:
            break
        rows = logits_fn([s[0] for s in active])
        pool = []
        full = []
        ai = 0
        for prefix, score, done, v in slots:
            if done:
                pool.append((prefix, score, True, -1))
                full.append((score, prefix + [BO.EOS]))
                continue
            row = [float(x) for x in rows[ai]]
            ai += 1
            lse = BO._lse([row[c] for c in range(len(row)) if allowed is None or allowed[c]])
            if v not in edges:
                edges[v] = {int(edge_class[j]): int(edge_child[j]) for j in range(int(first_edge[v]), int(first_edge[v + 1]))}
            kids = edges[v] if i + 1 < num_steps else {}
            order = [c for c in BO.row_order(row, allowed) if (c == BO.EOS and terminal[v]) or c in kids]
            full += [(score + (row[c] - lse), prefix + [c]) for c in order]
            for c in order[:K]:
                child = score + (row[c] - lse)
                if c == BO.EOS:
                    pool.append((prefix, child, True, -1))
                else:
                    pool.append((prefix + [c], child, False, kids[c]))
        if pools is not None:
            pools.append(sorted((f for f in full if not math.isnan(f[0]) and f[0] != BO.NEG_INF), key=lambda f: -f[0]))
        pool = [p for p in pool if p[1] != BO.NEG_INF]
        slots = sorted(pool, key=lambda p: BO.rank_key(p[1]))[:K]
    return [(p, s) for p, s, _, _ in slots]


def ranked_words(logits_fn, words: Sequence[Sequence[int]], num_steps: int, allowed=None):
    """The distinct words that fit (at most num_steps - 1 characters) with their log-likelihoods, best first."""
    out = {tuple(w): BO.sequence_logprob(logits_fn, list(w), num_steps, allowed) for w in words if len(w) < num_steps}
    return sorted(([list(w), s] for w, s in out.items()), key=lambda p: -p[1])
