"""Lexicons for constrained beam search (parseq_beam_search_lexicon): the words compiled to a prefix trie in the CSR
layout of parseq_lexicon_desc, uploaded once per engine."""
from __future__ import annotations

import weakref
from collections import deque
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .tokenizer import Tokenizer


def build_trie(rows: Sequence[Sequence[Sequence[int]]]):
    """A BFS-numbered prefix trie forest of class-id words: one tree per row, rooted at node r for row r.  Returns
    (first_edge int32 [V + 1], edge_class int32 [E], edge_child int32 [E], terminal uint8 [V]).  The numbering is
    breadth-first over the forest (the roots first, then each node's children in class order), so every child is
    numbered above its parent and each node's edge classes are strictly increasing.  Duplicate words share their node."""
    tries: List[Dict] = []
    for words in rows:
        root: Dict = {}
        for w in words:
            node = root
            for c in w:
                node = node.setdefault(int(c), {})
            node[-1] = True                               # key -1 marks the end of a word (classes are >= 1)
        tries.append(root)
    first, cls, child, term = [0], [], [], []
    queue = deque(tries)
    nxt = len(tries)                                      # the next free node number
    while queue:
        node = queue.popleft()
        term.append(1 if node.get(-1) else 0)
        for c in sorted(k for k in node if k >= 0):
            cls.append(c)
            child.append(nxt)
            nxt += 1
            queue.append(node[c])
        first.append(len(cls))
    return (np.asarray(first, dtype=np.int32), np.asarray(cls, dtype=np.int32), np.asarray(child, dtype=np.int32),
            np.asarray(term, dtype=np.uint8))


def lexicon_rows(candidates, batch: Optional[int] = None) -> Tuple[bool, List[Sequence[str]]]:
    """The structure checks of a word list or of one list per image, with pack_candidates' exceptions and messages:
    (shared, rows); for a shared list rows is [candidates].  `batch` (when known) is the number of images."""
    if isinstance(candidates, str) or not isinstance(candidates, (list, tuple)) or len(candidates) == 0:
        raise TypeError("candidates must be a non-empty list of strings, or one non-empty list of strings per image")
    if all(isinstance(c, str) for c in candidates):
        return True, [candidates]
    rows = list(candidates)
    if batch is not None and len(rows) != batch:
        raise ValueError(f"candidates has {len(rows)} lists for {batch} images")
    for b, r in enumerate(rows):
        if isinstance(r, str) or not isinstance(r, (list, tuple)) or len(r) == 0 or not all(isinstance(s, str) for s in r):
            raise TypeError(f"candidates of image {b} must be a non-empty list of strings")
    return False, rows


def check_words(tokenizer: Tokenizer, words, max_label_length: int, num_classes: int):
    """pack_candidates' character and length checks of a set of words."""
    words = sorted(words)
    unknown = sorted({ch for s in words for ch in s
                      if ch not in tokenizer._stoi or not 1 <= tokenizer._stoi[ch] < num_classes})
    if unknown:
        raise ValueError(f"candidate characters not in charset_train: {''.join(unknown)!r}")
    too_long = [s for s in words if len(s) > max_label_length]
    if too_long:
        raise ValueError(f"candidate {too_long[0]!r} has {len(too_long[0])} characters, more than max_label_length = "
                         f"{max_label_length}")


class Lexicon:
    """A compiled lexicon: the distinct words of one shared list, or of one list per image, as a BFS-numbered prefix trie
    (a forest with one root per distinct per-image list).  `roots` is None for a shared lexicon (node 0), else int32 [N]:
    image b starts at node roots[b].  The host arrays are kept; each engine uploads them once, on first use (a model
    moved to another device builds a new engine, and with it a new upload)."""

    def __init__(self, tokenizer: Tokenizer, candidates, max_label_length: int, num_classes: int):
        shared, rows = lexicon_rows(candidates)
        check_words(tokenizer, {s for r in rows for s in r}, max_label_length, num_classes)
        # what the trie's class ids mean and how long a word may be: beam_search refuses a model that differs
        self.charset = "".join(tokenizer._itos[1:tokenizer.bos_id])
        self.num_classes = num_classes
        self.max_label_length = max_label_length
        distinct: Dict[frozenset, int] = {}
        row_of = [distinct.setdefault(frozenset(r), len(distinct)) for r in rows]
        self.words: List[List[str]] = [sorted(ws) for ws in distinct]          # each tree's words
        ids = [[tokenizer._tok2ids(s) for s in ws] for ws in self.words]
        self.first_edge, self.edge_class, self.edge_child, self.terminal = build_trie(ids)
        self.roots: Optional[torch.Tensor] = None if shared else torch.tensor(row_of, dtype=torch.int32)
        self._handles = weakref.WeakKeyDictionary()       # Engine -> its device copy (freed with either side)

    @property
    def num_nodes(self) -> int:
        return int(self.terminal.shape[0])

    @property
    def num_edges(self) -> int:
        return int(self.edge_class.shape[0])

    @property
    def nbytes(self) -> int:
        """Device bytes of one upload (parseq_lexicon_create)."""
        return 4 * (self.num_nodes + 1) + 8 * max(self.num_edges, 1) + self.num_nodes

    def roots_for(self, batch: int) -> Optional[torch.Tensor]:
        """The roots of a call on `batch` images (None: node 0 for all)."""
        if self.roots is None:
            return None
        if self.roots.shape[0] != batch:
            raise ValueError(f"candidates has {self.roots.shape[0]} lists for {batch} images")
        return self.roots

    def handle(self, engine):
        """This lexicon on `engine`'s device (uploaded on the first call for that engine)."""
        h = self._handles.get(engine)
        if h is None:
            h = engine.lexicon_create(self.first_edge, self.edge_class, self.edge_child, self.terminal,
                                      torch.cuda.current_stream(engine.device).cuda_stream)
            self._handles[engine] = h
        return h
