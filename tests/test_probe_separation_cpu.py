"""The probes of tests/probe_models.py separate what the error budgets cannot (no GPU).

For every probe, on the CPU: the fp32 stand-in (the probe's fp64 model with fp32 arithmetic, i.e. what a correct engine
looks like) is within 1/10 of the probe's tolerance, and each bug the probe covers moves its output by 10x the tolerance
or more, in every decoder output (AR with and without the cluster kernel's hi + lo operands, refinement, NAR, and the
log_softmax terms `score` returns for the AR pass's teacher-forced candidates) or in the outputs the probe lists for it (`Probe.moves`: a mask bug of the refinement cannot touch AR); every pass it leaves out
stays bit-identical, so the list cannot go stale.  And the
probes cover every bug the budget tests leave out: each (budget key, bug) pair of the EXCLUDED tables of
test_encoder_budget_cpu.py and test_decoder_budget_cpu.py is covered by some probe at that key, so an entry added there
without a probe fails here."""
import functools

import pytest
import torch

import probe_models as pm
from test_decoder_budget_cpu import EXCLUDED as DEC_EXCLUDED
from test_encoder_budget_cpu import EXCLUDED as ENC_EXCLUDED

PROBES = pm.all_probes()
DEC_PASSES = [("ar", False), ("ar", True), ("refine", False), ("nar", False)]


def _id(entry):
    fn, args = entry
    return _probe(fn, args).name


@functools.lru_cache(maxsize=None)
def _probe(fn, args):
    return fn(*args)


def _err(a, b):
    return (a.double() - b.double()).abs().max().item()


def _outputs(p, **kw):
    if not p.decoder:
        return {"encoder": p.expected(**kw)}
    mem = p.memory()
    out = {f"{ps}{'-cluster' if cl else ''}": p.expected(pass_=ps, cluster=cl, memory=mem, **kw) for ps, cl in DEC_PASSES}
    out["score"] = pm.teacher_forced_terms(out["ar"], p.forced)
    return out


@functools.lru_cache(maxsize=None)
def _reference(fn, args):
    return _outputs(_probe(fn, args))


@pytest.mark.parametrize("entry", PROBES, ids=[_id(e) for e in PROBES])
def test_probe_is_finite_and_its_memory_exact(entry):
    p = _probe(*entry)
    for k, v in _reference(*entry).items():
        assert torch.isfinite(v).all(), k
    if p.decoder:
        mem = p.memory()
        assert torch.equal(mem.abs(), torch.ones_like(mem))


@pytest.mark.parametrize("entry", PROBES, ids=[_id(e) for e in PROBES])
def test_fp32_stand_in_is_within_a_tenth_of_the_tolerance(entry):
    p = _probe(*entry)
    got = _outputs(p, accum=torch.float32)
    for k, ref in _reference(*entry).items():
        e = _err(got[k], ref)
        print(f"{p.name} {k}: fp32 stand-in {e:.2e}  tolerance {p.tol:.0e}")
        assert e <= p.tol / 10, (k, e)


@pytest.mark.parametrize("entry", PROBES, ids=[_id(e) for e in PROBES])
def test_every_covered_bug_is_10x_over_the_tolerance(entry):
    p = _probe(*entry)
    ref = _reference(*entry)
    for bug in sorted({b for b, _ in p.covers}):
        got = _outputs(p, bug=bug)
        moved = p.moves.get(bug, tuple(ref))
        assert set(moved) <= set(ref), (bug, moved)
        for k in ref:
            e = _err(got[k], ref[k])
            print(f"{p.name} {bug} {k}: {e:.2e} = {e / p.tol:.0f}x the tolerance")
            if k in moved:
                assert e >= 10 * p.tol, (bug, k, e)
            else:
                assert torch.equal(got[k], ref[k]), (bug, k, "moves a pass the probe does not list", e)


def test_every_excluded_bug_is_covered_by_a_probe():
    covered = {c for e in PROBES for c in _probe(*e).covers}
    missing = [(bug, key) for table in (ENC_EXCLUDED, DEC_EXCLUDED) for key, bugs in table.items() for bug in bugs
               if (bug, key) not in covered]
    assert not missing, missing


def test_gelu_points_straddle_the_tanh_form():
    """Enough points, on both sides of 0, where only the tanh GELU changes the bf16 hidden value."""
    x, s = pm.gelu_points()
    assert x.numel() >= 100 and (x < 0).any() and (x > 0).any()
    assert set(s.tolist()) <= {-1.0, 1.0}
