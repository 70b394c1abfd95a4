"""CPU: lexicon-constrained beam search (parseq_beam_search_lexicon).  The fp64 rule (tests/lexicon_oracle.py) on
hand-built logits, its exhaustiveness when the beam is at least as wide as the lexicon, the trie builder's layout, the
Python checks, and the C ABI's host checks of malformed lexicons through the library built on this machine."""
import ctypes as C
import math
import random

import numpy as np
import pytest
import torch

import beam_oracle as BO
import lexicon_oracle as LO

INF = float("inf")


def random_ar_fn(C_, seed, sigma=2.0):
    def fn(prefixes):
        rows = []
        for p in prefixes:
            rng = random.Random(hash((seed, tuple(p))) & 0xffffffff)
            rows.append([rng.gauss(0.0, sigma) for _ in range(C_)])
        return rows
    return fn


def trie(words):
    from parseq_b200.lexicon import build_trie
    return build_trie([words])


# ---------------------------------------------------------------- the rule
@pytest.mark.parametrize("seed", range(6))
def test_wide_beam_is_exhaustive_over_the_lexicon(seed):
    """K >= |W| and no pruning: every word that fits comes back, ranked by its log-likelihood."""
    rng = random.Random(seed)
    C_, S = 6, 5                                             # 5 characters, num_steps 5: words of up to 4 characters
    words = {tuple(rng.randrange(1, C_) for _ in range(rng.randrange(0, 6))) for _ in range(12)}
    words |= {(), (1,), (1, 2), (1, 2, 3)}                    # the empty word and words that are prefixes of others
    words = sorted(words)
    fn = random_ar_fn(C_, seed)
    fit = LO.ranked_words(fn, words, S)
    K = min(16, len(words))
    assert len(fit) <= K
    got = LO.lexicon_beam_search(fn, K, S, *trie(words))
    assert [p for p, _ in got] == [p for p, _ in fit]
    for (_, a), (_, b) in zip(got, fit):
        assert a == pytest.approx(b, abs=1e-12)
    assert all(len(p) < S for p, _ in got)                    # too-long words never appear


def test_lse_is_over_the_whole_row_not_the_children():
    row = [0.5, 2.0, 1.0, -1.0]
    got = LO.lexicon_beam_search(lambda ps: [row for _ in ps], 4, 3, *trie([(2,)]))
    lse = math.log(sum(math.exp(v) for v in row))
    assert got == [([2], pytest.approx((1.0 - lse) + (0.5 - lse)))]


def test_allowlist_and_minus_inf_prune_children_but_eos_stays():
    row = [0.0, 1.0, -INF, 3.0]
    fn = lambda ps: [row for _ in ps]                                       # noqa: E731
    f = trie([(), (1,), (2,), (3,)])
    got = LO.lexicon_beam_search(fn, 4, 3, *f, allowed=[True, True, True, False])
    assert sorted(tuple(p) for p, _ in got) == [(), (1,)]                   # 2 is -inf, 3 is masked
    lse = math.log(1 + math.exp(1.0))                                       # allowed classes 0, 1 (2 is -inf)
    assert dict((tuple(p), s) for p, s in got)[()] == pytest.approx(0.0 - lse)


def test_no_word_reachable_gives_no_hypothesis():
    got = LO.lexicon_beam_search(lambda ps: [[0.0, 1.0, 2.0] for _ in ps], 3, 2, *trie([(1, 2)]))
    assert got == []                                                        # "12" needs 3 positions


def test_k1_follows_the_best_child_not_the_best_class():
    row = [0.0, 5.0, 1.0]
    got = LO.lexicon_beam_search(lambda ps: [row for _ in ps], 1, 4, *trie([(2, 2)]))
    assert [p for p, _ in got] == [[2, 2]]


# ---------------------------------------------------------------- the trie builder
def test_trie_layout_bfs_sorted_terminal():
    from parseq_b200.lexicon import build_trie
    first, cls, child, term = build_trie([[(2, 1), (1,), (), (2, 1), (2, 3)]])
    # node 0 root ("" is a word), children 1 (class 1) and 2 (class 2); node 2's children 3 (class 1) and 4 (class 3)
    assert first.tolist() == [0, 2, 2, 4, 4, 4]
    assert cls.tolist() == [1, 2, 1, 3] and child.tolist() == [1, 2, 3, 4]
    assert term.tolist() == [1, 1, 0, 1, 1]
    assert first.dtype == np.int32 and cls.dtype == np.int32 and child.dtype == np.int32 and term.dtype == np.uint8


def test_trie_forest_has_one_root_per_row_and_children_above_parents():
    from parseq_b200.lexicon import build_trie
    rows = [[(1, 2), (3,)], [(1,)], [()]]
    first, cls, child, term = build_trie(rows)
    V = term.shape[0]
    assert V == 3 + 4
    assert term[:3].tolist() == [0, 0, 1]                   # roots 0, 1, 2; only row 2 spells ""
    for v in range(V):
        e = range(first[v], first[v + 1])
        assert all(child[j] > v for j in e)
        assert list(cls[list(e)]) == sorted(set(cls[list(e)]))

    def words_of(root):
        out, stack = [], [(root, ())]
        while stack:
            v, p = stack.pop()
            if term[v]:
                out.append(p)
            stack += [(int(child[j]), p + (int(cls[j]),)) for j in range(first[v], first[v + 1])]
        return sorted(out)
    assert [words_of(r) for r in range(3)] == [[(1, 2), (3,)], [(1,)], [()]]


def test_compile_lexicon_dedups_and_checks_like_score():
    from parseq_b200.factory import create_model
    m = create_model("parseq-tiny")
    lex = m.compile_lexicon(["ab", "a", "ab", ""])
    assert lex.roots is None and lex.words == [["", "a", "ab"]]
    assert lex.num_nodes == 3 and lex.num_edges == 2 and lex.terminal.tolist() == [1, 1, 1]
    per = m.compile_lexicon([["a", "b"], ["b", "a"], ["c"]])
    assert per.roots.tolist() == [0, 0, 1] and per.words == [["a", "b"], ["c"]]
    with pytest.raises(ValueError, match="3 lists for 2 images"):
        per.roots_for(2)
    for bad, exc, msg in (("abc", TypeError, "non-empty list"), ([], TypeError, "non-empty list"),
                          ([["a"], []], TypeError, "image 1"), (["aé"], ValueError, "not in charset_train"),
                          (["x" * 26], ValueError, "more than max_label_length")):
        with pytest.raises(exc, match=msg):
            m.compile_lexicon(bad)


def test_beam_search_rejects_bad_lexicons_before_the_engine():
    from parseq_b200.factory import create_model
    m = create_model("parseq-tiny")
    x = torch.zeros(2, 3, 32, 128)
    with pytest.raises(ValueError, match="3 lists for 2 images"):
        m.beam_search(x, 4, lexicon=[["a"], ["b"], ["c"]])
    with pytest.raises(ValueError, match="not in charset_train"):
        m.lexicon_decode(x, ["é"], beam_width=4)
    with pytest.raises(ValueError, match="beam_width"):
        m.lexicon_decode(x, ["a"], beam_width=0)
    with pytest.raises(TypeError, match="compiled Lexicon serves the beam search only"):
        m.lexicon_decode(x, m.compile_lexicon(["a"]))


# ---------------------------------------------------------------- the C ABI's host checks
def _desc(first, cls, child, term, V=None, E=None):
    from parseq_b200.engine import LexiconDescC
    arrs = [np.ascontiguousarray(first, dtype=np.int32), np.ascontiguousarray(cls, dtype=np.int32),
            np.ascontiguousarray(child, dtype=np.int32), np.ascontiguousarray(term, dtype=np.uint8)]
    d = LexiconDescC(len(term) if V is None else V, len(cls) if E is None else E, *(a.ctypes.data for a in arrs))
    return d, arrs


GOOD = ([0, 2, 3, 3, 3], [1, 5, 2], [1, 2, 3], [0, 1, 0, 1])   # the words (1) and (1, 2); node 2 (class 5) is no word

BAD = [
    ("no nodes", dict(V=0), "num_nodes"),
    ("negative edges", dict(E=-1), "num_edges"),
    ("first_edge not ending at E", dict(first=[0, 2, 3, 3, 2]), "first_edge must start at 0 and end"),
    ("first_edge not starting at 0", dict(first=[1, 2, 3, 3, 3]), "first_edge must start at 0"),
    ("non-monotone first_edge", dict(first=[0, 2, 1, 3, 3]), "not monotone"),
    ("class 0 (EOS)", dict(cls=[0, 5, 2]), "outside 1..94"),
    ("class C", dict(cls=[1, 95, 2]), "outside 1..94"),
    ("unsorted classes", dict(cls=[5, 1, 2]), "not strictly increasing"),
    ("duplicate classes", dict(cls=[5, 5, 2]), "not strictly increasing"),
    ("child == parent", dict(child=[0, 2, 3]), "has child 0"),
    ("child below parent", dict(child=[1, 2, 1]), "has child 1"),
    ("child out of range", dict(child=[1, 2, 4]), "has child 4"),
]


@pytest.mark.parametrize("name,change,msg", BAD, ids=[b[0] for b in BAD])
def test_lexicon_check_rejects_malformed_lexicons(lib, name, change, msg):
    from parseq_b200.config import make_config
    from parseq_b200.engine import config_c
    cfg = config_c(make_config("parseq"))
    first, cls, child, term = (change.get(k, v) for k, v in zip(("first", "cls", "child", "term"), GOOD))
    d, keep = _desc(first, cls, child, term, V=change.get("V"), E=change.get("E"))
    assert lib.parseq_lexicon_check(C.byref(cfg), C.byref(d)) == -1
    assert msg in lib.parseq_last_error().decode(), lib.parseq_last_error().decode()


def test_lexicon_check_bounds_the_longest_path(lib):
    from parseq_b200.config import make_config
    from parseq_b200.engine import config_c
    from parseq_b200.lexicon import build_trie
    cfg = make_config("parseq")                                   # max_label_length 25
    for n, ok in ((25, True), (26, False)):
        # a chain of n edges with a short branch: the DAG check follows the longest path, not the first one
        d, keep = _desc(*build_trie([[(1,) * n, (2,)]]))
        rc = lib.parseq_lexicon_check(C.byref(config_c(cfg)), C.byref(d))
        assert rc == (0 if ok else -1), lib.parseq_last_error().decode()
        if not ok:
            assert "more than max_label_length = 25" in lib.parseq_last_error().decode()
    # a DAG whose node 2 is reached by a path of 1 edge (0 -> 2) and one of 2 (0 -> 1 -> 2), then a chain of 24 edges
    # to node 26: the longest path has 26 edges
    first = [0, 2] + list(range(3, 28)) + [27]
    cls = [1, 2, 3] + [1] * 24
    child = [1, 2, 2] + list(range(3, 27))
    term = [0] * 26 + [1]
    d, keep = _desc(first, cls, child, term)
    assert lib.parseq_lexicon_check(C.byref(config_c(cfg)), C.byref(d)) == -1     # 0 -> 1 -> 2 -> ... 26: 26 edges
    cfg.max_label_length = 26
    assert lib.parseq_lexicon_check(C.byref(config_c(cfg)), C.byref(d)) == 0


def test_lexicon_check_accepts_compiled_lexicons(lib):
    from parseq_b200.config import make_config
    from parseq_b200.engine import config_c, lexicon_desc
    from parseq_b200.factory import create_model
    m = create_model("parseq")
    cfg = config_c(make_config("parseq"))
    for words in (["hello", "help", "", "~" * 25], [[""], ["ab", "abc"], ["z"]]):
        lex = m.compile_lexicon(words)
        d = lexicon_desc(lex.first_edge, lex.edge_class, lex.edge_child, lex.terminal)
        assert lib.parseq_lexicon_check(C.byref(cfg), C.byref(d)) == 0, lib.parseq_last_error().decode()
    d, keep = _desc([0, 0], [], [], [1])                          # the lexicon {""}: one node, no edges
    assert lib.parseq_lexicon_check(C.byref(cfg), C.byref(d)) == 0


# ---------------------------------------------------------------- goldens (tests/make_golden_lexicon.py)
def test_goldens_load_stay_small_and_hold_words_of_their_lexicons():
    import glob
    import os
    from make_golden_beam import GOLDEN_FILE_LIMIT, golden_state_dict
    from make_golden_lexicon import CASES
    from make_golden_long import make_config_long
    from parseq_b200.tokenizer import Tokenizer
    from parseq_b200.weights import state_dict_digest
    paths = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lexicon", "lx_*.pt")))
    assert len(paths) == len(CASES)
    for path in paths:
        assert os.path.getsize(path) < GOLDEN_FILE_LIMIT, path
        blob = torch.load(path, weights_only=False)
        extra = {} if blob["experiment"] == "vitstr" else {"dec_depth": blob["dec_depth"]}
        cfg = make_config_long(blob["experiment"], blob["max_label_length"], blob["n_extra"], **extra)
        assert state_dict_digest(golden_state_dict(cfg, blob["weight_seed"], blob["sharp"])) == blob["sd_digest"], path
        tok = Tokenizer(cfg.charset_train)
        lex = blob["lexicon"]
        rows = lex if isinstance(lex[0], list) else [lex] * blob["batch"]
        for b, im in enumerate(blob["images"]):
            s = im["scores"]
            assert 1 <= len(im["ids"]) <= blob["beam_width"] and bool((s[:-1] >= s[1:]).all())
            allow = None if blob["allowlist"] is None else blob["allowlist"][b]
            for p in im["ids"]:
                w = tok._ids2tok(p, True)
                assert w in rows[b] and len(w) <= blob["max_label_length"], (path, b, w)
                assert allow is None or set(w) <= set(allow)
