"""CPU: character maps for given text (parseq_score_args.attn_maps, parseq_beam_args.attn_maps, score / beam_search /
lexicon_decode(return_attention=True) and locate(text=)).  The argument checks refuse, or accept, before a handle or a
device is needed; the fp64 rounding-point rule of tests/attn_maps_reference.py, fed a candidate's teacher-forced ids,
agrees with the maps the reference's own modules record (tests/golden/alignment, tests/make_golden_alignment.py)."""
import ctypes as C
import os

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from parseq_b200.engine import load_library
    try:
        return load_library()
    except (RuntimeError, OSError) as e:
        pytest.skip(str(e))


def _system(experiment="parseq", **kw):
    from parseq_b200.factory import create_model
    return create_model(experiment, **kw)


def _score_args(maps_ptr):
    from parseq_b200.engine import ScoreArgsC
    per = (C.c_int32 * 1)(2)
    tg = (C.c_int32 * 52)()
    tg[0], tg[1] = 5, 0               # "x" + EOS
    tg[26] = 0                        # "" + EOS
    ln = (C.c_int32 * 2)(1, 0)
    return ScoreArgsC(1, 2, C.addressof(per), C.addressof(tg), C.addressof(ln), maps_ptr), (per, tg, ln)


def test_struct_fields_are_appended_last():
    from parseq_b200.engine import BeamArgsC, ScoreArgsC
    assert ScoreArgsC._fields_[-1] == ("attn_maps", C.c_void_p)
    assert [n for n, _ in ScoreArgsC._fields_[:-1]] == ["batch", "num_candidates", "per_image", "targets", "lengths"]
    assert BeamArgsC._fields_[-1] == ("attn_maps", C.c_void_p)
    assert [n for n, _ in BeamArgsC._fields_[:-1]] == ["batch", "beam_width", "max_length", "class_mask"]


def test_score_check_accepts_maps_for_parseq(lib):
    from parseq_b200.config import make_config
    from parseq_b200.engine import config_c
    buf = (C.c_float * 4)()
    a, keep = _score_args(C.addressof(buf))
    assert lib.parseq_score_check(C.byref(config_c(make_config("parseq"))), C.byref(a)) == 0
    a, keep = _score_args(None)
    assert lib.parseq_score_check(C.byref(config_c(make_config("vitstr"))), C.byref(a)) == 0


def test_score_check_rejects_maps_for_vitstr(lib):
    from parseq_b200.config import make_config
    from parseq_b200.engine import config_c
    buf = (C.c_float * 4)()
    a, keep = _score_args(C.addressof(buf))
    assert lib.parseq_score_check(C.byref(config_c(make_config("vitstr"))), C.byref(a)) == -2
    assert "ViTSTR has no decoder cross-attention" in lib.parseq_last_error().decode()


def test_score_check_still_checks_targets_with_maps(lib):
    from parseq_b200.config import make_config
    from parseq_b200.engine import config_c
    buf = (C.c_float * 4)()
    a, keep = _score_args(C.addressof(buf))
    keep[1][1] = 7                     # candidate 0 loses its EOS
    assert lib.parseq_score_check(C.byref(config_c(make_config("parseq"))), C.byref(a)) == -1
    assert "no EOS" in lib.parseq_last_error().decode()


@pytest.mark.parametrize("call", ["score", "beam_search", "lexicon_decode", "lexicon_decode_beam"])
def test_vitstr_refuses_maps(call):
    m = _system("vitstr")
    x = torch.zeros((1, 3, 224, 224))
    with pytest.raises(NotImplementedError, match="no decoder cross-attention"):
        if call == "score":
            m.score(x, ["a"], return_attention=True)
        elif call == "beam_search":
            m.beam_search(x, 2, return_attention=True)
        elif call == "lexicon_decode":
            m.lexicon_decode(x, ["a"], return_attention=True)
        else:
            m.lexicon_decode(x, ["a"], beam_width=2, return_attention=True)
    with pytest.raises(NotImplementedError):
        m.locate(x, text="a")


@pytest.mark.parametrize("text, msg", [
    (["a"], "one string or a list of 2 strings"),
    (["a", "b", "c"], "one string or a list of 2 strings"),
    (["a", 3], "one string or a list of 2 strings"),
    (7, "one string or a list of 2 strings"),
])
def test_locate_text_rejects_bad_text(text, msg):
    m = _system("parseq")
    with pytest.raises(ValueError, match=msg):
        m.locate(torch.zeros((2, 3, 32, 128)), text=text)


@pytest.mark.parametrize("kw", [dict(max_length=5), dict(allowlist="abc"), dict(orientations=[0, 180]),
                                dict(min_confidence=0.5)], ids=["max_length", "allowlist", "orientations",
                                                                "min_confidence"])
def test_locate_text_rejects_conflicting_options(kw):
    m = _system("parseq")
    with pytest.raises(ValueError, match="text fixes the characters"):
        m.locate(torch.zeros((1, 3, 32, 128)), text="a", **kw)


@pytest.mark.parametrize("text", ["café", "a一", "x" * 26], ids=["accent", "cjk", "too_long"])
def test_locate_text_rejects_what_score_rejects(text):
    m = _system("parseq")
    x = torch.zeros((1, 3, 32, 128))
    with pytest.raises(ValueError) as by_score:
        m.score(x, [text], return_attention=True)
    with pytest.raises(ValueError) as by_locate:
        m.locate(x, text=text)
    assert str(by_locate.value) == str(by_score.value)


# ---- the fp64 rule against the reference's own maps (tests/golden/alignment, tests/make_golden_alignment.py) ---------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "alignment")
GOLDENS = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.endswith(".pt")) if os.path.isdir(GOLDEN) else []


def test_golden_set_covers_the_cases():
    kinds = set()
    for name in GOLDENS:
        b = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
        kinds.add((b["experiment"], b["dec_depth"], b["max_label_length"], b["n_extra"], b["sharp"] > 0))
        assert b["maps"].shape[0] == sum(len(c) + 1 for r in b["candidates"] for c in r)
    assert ("parseq", 1, 25, 0, True) in kinds and ("parseq-tiny", 1, 25, 2906, True) in kinds
    assert ("parseq", 2, 25, 0, True) in kinds and ("parseq", 1, 63, 0, True) in kinds
    assert ("parseq-patch16-224", 1, 25, 0, True) in kinds


@pytest.mark.parametrize("name", GOLDENS)
def test_rounding_point_rule_agrees_with_goldens(name):
    """tests/attn_maps_reference.py fed each candidate's teacher-forced ids and the fp64 oracle's memory: rows 0..n of
    every candidate within GOLDEN_BOUNDS of the reference's maps."""
    from attn_maps_reference import GOLDEN_BOUNDS, MapsReference, excess, format_stats, map_stats
    from dec_depth_oracle import DepthOracle
    from make_golden_alignment import golden_case
    blob, cfg, sd, x, targets, lengths, _ = golden_case(name)
    mem = DepthOracle(cfg, sd, "fp64").encode(x)
    ref = MapsReference(cfg, sd)
    rows, m = [], 0
    for b, cands in enumerate(blob["candidates"]):
        for _ in cands:
            n = int(lengths[m])
            rows.append(ref.ar(mem[b:b + 1], targets[m:m + 1])[0, :n + 1])
            m += 1
    got = torch.cat(rows)
    s = map_stats(got, blob["maps"])
    print(format_stats(name, s))
    assert max(excess(s, GOLDEN_BOUNDS).values()) <= 1.0, s
