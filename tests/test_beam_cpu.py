"""CPU: the fp64 beam-search rule of parseq_beam_search (tests/beam_oracle.py) on hand-built logits, its exactness
against exhaustive enumeration where the beam holds every prefix, and the argument checks of the Python layer."""
import math
import random

import pytest
import torch

import beam_oracle as BO

NAN, INF = float("nan"), float("inf")


def table_fn(table):
    """logits_fn whose row depends only on the prefix length (ViTSTR-like) or on the prefix itself (dict)."""
    def fn(prefixes):
        return [table[tuple(p)] if isinstance(table, dict) else table[len(p)] for p in prefixes]
    return fn


def random_ar_fn(C, seed):
    """A deterministic function of the whole prefix: an AR model stand-in."""
    def fn(prefixes):
        rows = []
        for p in prefixes:
            rng = random.Random(hash((seed, tuple(p))) & 0xffffffff)
            rows.append([rng.gauss(0.0, 2.0) for _ in range(C)])
        return rows
    return fn


@pytest.mark.parametrize("seed", range(5))
def test_beam_equals_exhaustive_enumeration_when_it_holds_every_prefix(seed):
    # 3 characters, max_label_length 2 (num_steps 3): K = 16 keeps every prefix until the last step, so the beam is exact
    fn = random_ar_fn(4, seed)
    beams = BO.beam_search(fn, 16, 3)
    ex = BO.exhaustive(fn, 4, 3)[:16]
    assert [p for p, _ in beams] == [p for p, _ in ex]
    for (_, a), (_, b) in zip(beams, ex):
        assert a == pytest.approx(b, abs=1e-12)


def test_scores_are_the_teacher_forced_log_likelihood():
    fn = random_ar_fn(6, 7)
    for prefix, score in BO.beam_search(fn, 5, 4):
        assert score == pytest.approx(BO.sequence_logprob(fn, prefix, 4), abs=1e-12)


def test_k1_is_greedy():
    fn = random_ar_fn(6, 3)
    (prefix, _), = BO.beam_search(fn, 1, 5)
    greedy = []
    for _ in range(5):
        row = fn([greedy])[0]
        c = max(range(6), key=lambda j: (row[j], -j))
        if c == 0:
            break
        greedy.append(c)
    assert prefix == greedy


def test_row_order_nan_first_then_descending_ties_to_lower_class():
    row = [1.0, NAN, 3.0, 3.0, -INF, NAN, 0.5]
    assert BO.row_order(row) == [1, 5, 2, 3, 0, 6]
    assert BO.row_order(row, [True, False, True, False, True, True, True]) == [5, 2, 0, 6]


def test_ties_keep_pool_order():
    # two identical rows: the children of slot 0 come first in the pool, so they win the ties
    row = [0.0, 1.0, 1.0]
    beams = BO.beam_search(table_fn([row, row]), 2, 2)
    assert [p for p, _ in beams] == [[1, 1], [1, 2]]
    assert beams[0][1] == beams[1][1]


def test_nan_row_ranks_after_numbers():
    # the row after "1" holds a NaN: its LSE is NaN, so all its children are NaN and rank after the finite entries
    table = {(): [0.0, 2.0, 1.0], (1,): [0.0, NAN, 0.0], (2,): [3.0, 0.0, 0.0]}
    beams = BO.beam_search(table_fn(table), 5, 2)
    assert [math.isnan(s) for _, s in beams] == [False, False, False, False, True]
    assert beams[-1][0] == [1, 1]                     # the NaN logit expands first within its row
    # the NaN row's LSE is NaN, so every child of it is NaN
    assert all(math.isnan(s) for _, s in BO.beam_search(table_fn([[0.0, 1.0, NAN]]), 3, 1))


def test_minus_inf_and_masked_classes_never_expand():
    beams = BO.beam_search(table_fn([[0.0, -INF, 2.0, 1.0]]), 4, 1)
    assert sorted(p[0] if p else 0 for p, _ in beams) == [0, 2, 3]
    beams = BO.beam_search(table_fn([[0.0, 5.0, 2.0, 1.0]]), 4, 1, allowed=[True, False, True, False])
    assert [p for p, _ in beams] == [[2], []]
    # the LSE runs over the allowed classes only
    assert beams[0][1] == pytest.approx(2.0 - math.log(math.exp(0.0) + math.exp(2.0)), abs=1e-12)


def test_empty_allowlist_gives_the_empty_reading_with_score_zero():
    beams = BO.beam_search(random_ar_fn(5, 1), 4, 3, allowed=[False] * 5)
    assert beams == [([], 0.0)]


def test_finished_slots_are_carried_and_no_eos_runs_to_num_steps():
    # EOS is most likely at step 0 and never again: "" finishes at once and stays; the rest fill num_steps characters
    beams = BO.beam_search(table_fn([[5.0, 1.0, 0.0], [-INF, 1.0, 0.0], [-INF, 1.0, 0.0]]), 3, 3)
    assert beams[0] == ([], pytest.approx(5.0 - math.log(math.exp(5) + math.exp(1) + 1)))
    assert all(len(p) == 3 for p, _ in beams[1:])


def test_beam_width_validation():
    from parseq_b200.system import check_beam_width
    for bad in (0, 17, -1, 2.0, True, "3", None):
        with pytest.raises(ValueError):
            check_beam_width(bad)
    assert check_beam_width(1) == 1 and check_beam_width(16) == 16


def test_system_rejects_bad_beam_width_before_the_engine():
    from parseq_b200.factory import create_model
    m = create_model("parseq-tiny")
    with pytest.raises(ValueError, match="beam_width"):
        m.beam_search(torch.zeros(1, 3, 32, 128), beam_width=0)
    with pytest.raises(ValueError, match="beam_width"):
        m.model.beam_search(torch.zeros(1, 3, 32, 128), beam_width=17)


# ---------------------------------------------------------------- goldens (tests/make_golden_beam.py)
import glob  # noqa: E402
import os  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "beam")


def test_goldens_load_stay_small_and_match_their_weights():
    from make_golden_beam import CASES, GOLDEN_FILE_LIMIT, golden_state_dict
    from make_golden_long import make_config_long
    from parseq_b200.weights import state_dict_digest
    paths = sorted(glob.glob(os.path.join(GOLDEN, "bm_*.pt")))
    assert len(paths) == len(CASES)
    for path in paths:
        assert os.path.getsize(path) < GOLDEN_FILE_LIMIT, path
        blob = torch.load(path, weights_only=False)
        extra = {} if blob["experiment"] == "vitstr" else {"dec_depth": blob["dec_depth"]}
        cfg = make_config_long(blob["experiment"], blob["max_label_length"], blob["n_extra"], **extra)
        sd = golden_state_dict(cfg, blob["weight_seed"], blob["sharp"])
        assert state_dict_digest(sd) == blob["sd_digest"], path
        L = blob["max_label_length"] + 1
        assert len(blob["images"]) == blob["batch"]
        for im in blob["images"]:
            s = im["scores"]
            assert 1 <= len(im["ids"]) <= blob["beam_width"] and len(s) == len(im["ids"])
            assert bool((s[:-1] >= s[1:]).all())
            assert all(len(p) <= L and all(1 <= c < cfg.num_classes for c in p) for p in im["ids"])
            assert len(im["prune_margins"]) >= 1 and bool((im["prune_margins"] >= 0).all())
