"""GPU: lexicon-constrained beam search (parseq_beam_search_lexicon; `beam_search(lexicon=)`, `lexicon_decode(beam_width=)`).

Every hypothesis is a word of the image's lexicon that ended with EOS.  Its score is the sum of log_softmax of the logits
the greedy chain of separate kernels (ar_kernel 0, no refinement) computes when it is teacher-forced along the word: the
lexicon step reads the same head output, so only the fp32 rounding of the log-sum-exp differs.  It also agrees with
`score()` of the word within the per-term bound of tests/test_gpu_beam.py.  With a beam at least as wide as the lexicon
the search is exhaustive.  Hypotheses and score bits do not depend on the rest of the call."""
import random

import numpy as np
import pytest
import torch

from test_gpu_beam import LSE_REL, TERM_MAX, _model, _same

pytestmark = pytest.mark.gpu


def _words(cs, n, seed, max_len, extra=()):
    rng = random.Random(seed)
    out = set(extra)
    while len(out) < n:
        out.add("".join(rng.choice(cs) for _ in range(rng.randint(1, max_len))))
    return sorted(out)


def _forced_logits(m, experiment, x, words, mll):
    """Teacher-forced logits [N, W, L, C] of every (image, word): the chain (ar_kernel 0) forced along c_1..c_n, EOS;
    ViTSTR's per-position logits do not depend on the word."""
    N, W, L = x.shape[0], len(words), mll + 1
    with torch.inference_mode():
        if experiment == "vitstr":
            lg = m.model.forward_tokens(x, None)
            return lg[:, None].expand(N, W, *lg.shape[1:])
        forced = torch.zeros((W, L), dtype=torch.int32)         # forced[:, j]: the id at position j (0 is BOS)
        for i, w in enumerate(words):
            ids = m.tokenizer._tok2ids(w)
            forced[i, 1:1 + len(ids)] = torch.tensor(ids, dtype=torch.int32)
        xs = x.repeat_interleave(W, 0)
        lg = m.model.forward(m.tokenizer, xs, mll, forced_ids=forced.repeat(N, 1).cuda())
    return lg.view(N, W, L, -1)


def _tf_score(m, lg, word, allowed=None):
    """(sum of the terms, tight bound): log_softmax over the allowed classes of rows 0..n at targets (c_1..c_n, EOS)."""
    t = m.tokenizer._tok2ids(word) + [0]
    rows = lg[:len(t)].double()
    if allowed is not None:
        rows = rows.masked_fill(~allowed[:rows.shape[1]].to(rows.device), float("-inf"))
    lse = torch.logsumexp(rows, -1)
    terms = rows.gather(1, torch.tensor(t, device=rows.device)[:, None])[:, 0] - lse
    return terms.sum().item(), (LSE_REL * (1 + lse.abs())).sum().item() + 1e-6 * len(t)


# ---------------------------------------------------------------- exhaustive search
EX_CASES = [("parseq", 25, 0, 1), ("parseq-tiny", 25, 2906, 1), ("parseq-tiny", 25, 16289, 1), ("parseq", 25, 0, 2),
            ("parseq", 63, 0, 1), ("vitstr", 25, 0, 1)]


@pytest.mark.parametrize("case", EX_CASES, ids=lambda c: f"{c[0]}-L{c[1] + 1}-C{95 + c[2]}-depth{c[3]}")
def test_wide_beam_returns_every_word_with_its_teacher_forced_score(case):
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    experiment, mll, n_extra, depth = case
    kw = {} if experiment == "vitstr" else {"refine_iters": 0}
    cfg, m = _model(experiment, mll, seed=101, n_extra=n_extra, dec_depth=depth, sharp=2.0, **kw)
    if experiment != "vitstr":
        m.model.set_engine_option("ar_kernel", 0)
    cs = charset(n_extra)
    a, b = cs[10:14], cs[-3:]
    # "" and words that are prefixes of each other, one of max_label_length characters, the rest random
    words = _words(cs, 16, 102, 6, extra=("", a[:1], a[:2], a, a + b, (b * mll)[:mll]))
    N = 3
    x = synth_images(cfg, N, 103).cuda()
    with torch.inference_mode():
        labels, scores = m.beam_search(x, 16, lexicon=words)
        ex_labels, ex_lp = m.lexicon_decode(x, words)
        _, sc = m.score(x, words, return_token_logprobs=True)
    lg = _forced_logits(m, experiment, x, words, mll)
    for b_ in range(N):
        assert sorted(labels[b_]) == words, b_
        s = scores[b_].double().cpu()
        assert bool((s[:-1] >= s[1:]).all())
        for k, w in enumerate(labels[b_]):
            ref, bound = _tf_score(m, lg[b_, words.index(w)], w)
            assert abs(s[k].item() - ref) <= bound, (b_, w, s[k].item(), ref)
            i = words.index(w)
            sref = sc[b_, i, :len(w) + 1].double().sum().item()
            assert abs(s[k].item() - sref) <= TERM_MAX * (len(w) + 1), (b_, w)
        # the top-1 is exhaustive lexicon_decode's pick wherever the runner-up is clear of both bounds
        gap = s[0].item() - s[1].item()
        if gap > TERM_MAX * (len(labels[b_][0]) + len(labels[b_][1]) + 2):
            assert labels[b_][0] == ex_labels[b_], b_


# ---------------------------------------------------------------- a large lexicon, per-image lexicons
def test_large_lexicon_hypotheses_are_words_best_first_with_tight_scores():
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", seed=111, sharp=2.0, refine_iters=0)
    m.model.set_engine_option("ar_kernel", 0)
    cs = charset(0)
    words = _words(cs, 20000, 112, 10)
    lex = m.compile_lexicon(words)
    N, K = 6, 8
    x = synth_images(cfg, N, 113).cuda()
    with torch.inference_mode():
        labels, scores = m.beam_search(x, K, lexicon=lex)
    wset = set(words)
    hyp = sorted({h for row in labels for h in row})
    lg = _forced_logits(m, "parseq", x, hyp, cfg.max_label_length)
    for b in range(N):
        assert len(labels[b]) == K and all(h in wset for h in labels[b])
        s = scores[b].double().cpu()
        assert bool((s[:-1] >= s[1:]).all())
        for k, h in enumerate(labels[b]):
            ref, bound = _tf_score(m, lg[b, hyp.index(h)], h)
            assert abs(s[k].item() - ref) <= bound, (b, h)
    # per-image lexicons of 50 words: each image's hypotheses come from its own list
    per = [_words(cs, 50, 120 + b, 8) for b in range(N)]
    with torch.inference_mode():
        labels, scores = m.beam_search(x, K, lexicon=per)
    for b in range(N):
        assert len(labels[b]) == K and all(h in per[b] for h in labels[b])


# ---------------------------------------------------------------- invariance
def test_hypotheses_do_not_depend_on_the_rest_of_the_call():
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", seed=131, sharp=2.0)
    m.model.set_engine_option("fuse_ln", 0)              # one encoder kernel regime at every batch size
    cs = charset(0)
    lex = m.compile_lexicon(_words(cs, 1000, 132, 8))
    x = synth_images(cfg, 1030, 133).cuda()
    with torch.inference_mode():
        ref = m.model.beam_search(x[:1], 5, lexicon=lex)
        for N, pos in ((7, 3), (130, 129), (1030, 0), (1030, 777)):
            xs = x[:N].clone()
            xs[pos] = x[0]
            out = m.model.beam_search(xs, 5, lexicon=lex)
            for r, o in zip(ref, out):
                assert _same(o[pos], r[0]), (N, pos)
        # the same words as one list per image: a forest with one tree, image b at its root
        per = m.compile_lexicon([lex.words[0]] * 7)
        out = m.model.beam_search(x[:7], 5, lexicon=per, roots=per.roots_for(7))
        for r, o in zip(ref, out):
            assert _same(o[0], r[0])
        m.model.set_engine_option("dec_chunk", 32)
        out = m.model.beam_search(x[:40], 5, lexicon=lex)
    for r, o in zip(ref, out):
        assert _same(o[0], r[0])
    rng = np.random.default_rng(134)
    u8 = torch.from_numpy(rng.integers(0, 256, (3, 32, 128, 3), dtype=np.uint8))
    xf = ((u8.permute(0, 3, 1, 2).to(torch.float32).div(255) - 0.5) / 0.5).cuda()
    crops = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).cuda() for h, w in ((20, 70), (64, 300), (32, 128))]
    with torch.inference_mode():
        a = m.model.beam_search(xf, 4, lexicon=lex)
        b = m.model.beam_search(u8.cuda(), 4, lexicon=lex)
        for p, q in zip(a, b):
            assert _same(p, q)
        c = m.beam_search(crops, 4, rotation=90, lexicon=lex)
        d = m.beam_search(m.preprocess(crops, 90), 4, lexicon=lex)
    assert c[0] == d[0] and _same(c[1], d[1])


def test_vitstr_hypotheses_do_not_depend_on_the_batch():
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, m = _model("vitstr", seed=141, sharp=2.0)
    lex = m.compile_lexicon(_words(charset(0), 500, 142, 8))
    x = synth_images(cfg, 70, 143).cuda()
    with torch.inference_mode():
        ref = m.model.beam_search(x[:1], 6, lexicon=lex)
        xs = x.clone()
        xs[69] = x[0]
        out = m.model.beam_search(xs, 6, lexicon=lex)
    for r, o in zip(ref, out):
        assert _same(o[69], r[0])


# ---------------------------------------------------------------- combinations and failure cases
@pytest.mark.parametrize("experiment", ["parseq", "vitstr"])
def test_allowlist_and_max_length_combine_with_the_lexicon(experiment):
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    kw = {} if experiment == "vitstr" else {"refine_iters": 0}
    cfg, m = _model(experiment, seed=151, sharp=2.0, **kw)
    if experiment != "vitstr":
        m.model.set_engine_option("ar_kernel", 0)
    cs = charset(0)
    words = _words(cs[:20], 12, 152, 6, extra=("", "0", "01", "012345678"))
    N = 4
    x = synth_images(cfg, N, 153).cuda()
    allow = ["0123456789", None, "0123456789abc", "01"]
    with torch.inference_mode():
        labels, scores = m.beam_search(x, 16, lexicon=words, allowlist=allow)
        short, _ = m.beam_search(x, 16, lexicon=words, max_length=3)
    lg = _forced_logits(m, experiment, x, words, cfg.max_label_length)
    mask = m.allowlist_mask(allow, N)
    bits = ((mask.cpu().long()[:, :, None] >> torch.arange(32)) & 1).bool().view(N, -1)
    for b in range(N):
        ok = [w for w in words if allow[b] is None or set(w) <= set(allow[b])]
        assert sorted(labels[b]) == ok, b
        for k, w in enumerate(labels[b]):
            ref, bound = _tf_score(m, lg[b, words.index(w)], w, bits[b])
            assert abs(scores[b, k].item() - ref) <= bound, (b, w)
        assert sorted(short[b]) == [w for w in words if len(w) <= 3]


@pytest.mark.parametrize("experiment", ["parseq", "vitstr"])
def test_nan_crop_stays_in_its_own_row(experiment):
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, m = _model(experiment, seed=161)
    lex = m.compile_lexicon(_words(charset(0), 200, 162, 8))
    x = synth_images(cfg, 5, 163).cuda()
    with torch.inference_mode():
        ref = m.model.beam_search(x, 4, lexicon=lex)
        xn = x.clone()
        xn[2] = float("nan")
        out = m.model.beam_search(xn, 4, lexicon=lex)
    keep = torch.tensor([0, 1, 3, 4], device="cuda")
    for r, o in zip(ref, out):
        assert _same(o[keep], r[keep])


def test_bad_inputs_raise_and_unreachable_words_give_none():
    from parseq_b200.engine import EngineError
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", seed=171)
    x = synth_images(cfg, 2, 172).cuda()
    with pytest.raises(ValueError, match="not in charset_train"):
        m.beam_search(x, 4, lexicon=["abc", "aé"])
    with pytest.raises(ValueError, match="more than max_label_length"):
        m.beam_search(x, 4, lexicon=["a" * 26])
    with pytest.raises(TypeError):
        m.beam_search(x, 4, lexicon=[])
    lex = m.compile_lexicon([["abc"], ["abcdef"]])
    with pytest.raises(EngineError, match="not a node"):
        m.model.beam_search(x, 4, lexicon=lex, roots=torch.tensor([0, 99], dtype=torch.int32))
    with torch.inference_mode():
        labels, lp = m.lexicon_decode(x, [["abc"], ["abcdef"]], beam_width=4)
        short = m.beam_search(x, 4, max_length=3, lexicon=[["abc"], ["abcdef"]])
    assert labels == ["abc", "abcdef"] and bool(torch.isfinite(lp).all())
    assert short[0] == [["abc"], []] and bool(torch.isneginf(short[1][1]).all())
    with torch.inference_mode():
        labels, lp = m.lexicon_decode(x[:1], ["abcd"], beam_width=2)
    assert labels == ["abcd"]


def test_no_lexicon_buffers_until_the_first_lexicon_call():
    """PARSeq-S at 95 classes, max_batch 512 and dec_chunk 128: 4 stages of 128 beam rows with ids_ld 32.  Per stage the
    plain beam holds ids 2 x 128 x 32, score / len / st 2 x 128 each, parent 128 (int32 / fp32) and the step's logits
    128 x 95 fp32; a lexicon adds the double-buffered nodes (2 x 128 int32 per stage) and the call's roots (int32 [N])."""
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", seed=181)
    x = synth_images(cfg, 16, 182).cuda()
    stages, rows = 4, 128
    plain_bytes = stages * 4 * (2 * rows * 32 + 3 * 2 * rows + rows + rows * cfg.num_classes)
    with torch.inference_mode():
        m.beam_search(x, 3)
        eng = m.model.engine()
        assert eng.debug_int("beam_bytes") == plain_bytes
        m.beam_search(x, 3, lexicon=_words(charset(0), 100, 183, 6))
        assert eng.debug_int("beam_bytes") == plain_bytes + stages * 4 * 2 * rows
        m.beam_search(x, 3, lexicon=[_words(charset(0), 20, 184 + b, 6) for b in range(16)])
        assert eng.debug_int("beam_bytes") == plain_bytes + stages * 4 * 2 * rows + 4 * 16
        m.beam_search(x, 3)
        assert eng.debug_int("beam_bytes") == plain_bytes + stages * 4 * 2 * rows + 4 * 16


# ---------------------------------------------------------------- per-image lexicons across groups and super-chunks
@pytest.mark.parametrize("experiment", ["parseq", "vitstr"])
def test_per_image_lexicons_across_groups_and_super_chunks(experiment):
    """Distinct 40-word lists for 130 images (PARSeq: dec_chunk 32, groups of 6 images at K = 5; both: max_batch 64, three
    super-chunks; ViTSTR: groups of 32).  Every image's hypotheses come from its own list, and the bits at group and
    super-chunk boundaries equal a one-image call with that image's list."""
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, m = _model(experiment, seed=191, sharp=2.0)
    m.model.set_engine_option("fuse_ln", 0)              # one encoder kernel regime at every batch size
    m.model.set_engine_option("max_batch", 64)
    if experiment != "vitstr":
        m.model.set_engine_option("dec_chunk", 32)
    cs = charset(0)
    N, K = 130, 5
    per = [_words(cs, 40, 1000 + b, 7) for b in range(N)]
    x = synth_images(cfg, N, 192).cuda()
    lex = m.compile_lexicon(per)
    assert len(lex.words) == N                           # distinct lists: one tree and one root each
    with torch.inference_mode():
        ids, lengths, scores = m.model.beam_search(x, K, lexicon=lex, roots=lex.roots_for(N))
        labels, _ = m.beam_search(x, K, lexicon=per)
    for b in range(N):
        assert len(labels[b]) == K and all(h in per[b] for h in labels[b]), b
    for b in (0, 5, 6, 31, 32, 63, 64, 65, 95, 127, 128, 129):
        one = m.compile_lexicon([per[b]])
        with torch.inference_mode():
            r = m.model.beam_search(x[b:b + 1], K, lexicon=one, roots=one.roots_for(1))
        for o, q in zip((ids, lengths, scores), r):
            assert _same(o[b], q[0]), b


def test_pinned_roots_may_be_reused_as_soon_as_the_call_returns():
    """The engine copies the roots on the host before it returns: overwriting a pinned roots buffer right after the call
    (with an out-of-range node) changes nothing."""
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", seed=195, sharp=2.0)
    cs = charset(0)
    N = 64
    per = [_words(cs, 30, 2000 + b, 7) for b in range(N)]
    lex = m.compile_lexicon(per)
    x = synth_images(cfg, N, 196).cuda()
    with torch.inference_mode():
        ref = m.model.beam_search(x, 4, lexicon=lex, roots=lex.roots_for(N).clone())
        pinned = lex.roots_for(N).clone().pin_memory()
        out = m.model.beam_search(x, 4, lexicon=lex, roots=pinned)
        pinned.fill_(1 << 30)
        torch.cuda.synchronize()
    for r, o in zip(ref, out):
        assert _same(o, r)


# ---------------------------------------------------------------- against the reference goldens (tests/make_golden_lexicon.py)
def test_lexicon_beams_match_reference_goldens():
    """The fp64 lexicon beams of the reference's own modules.  As tests/test_gpu_beam.py checks its goldens: every engine
    hypothesis equal to the golden's at its rank has a score within TERM_MAX per term, and where every pruning margin
    and the gaps to the neighbouring ranks exceed TERM_MAX times the terms the two scores do not share, the labels match
    rank by rank.  At least half of all golden hypotheses are checked."""
    import glob
    import os
    from make_golden_beam import distinct_terms, golden_state_dict
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import synth_images
    paths = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lexicon", "lx_*.pt")))
    assert paths
    total = checked = 0
    for path in paths:
        blob = torch.load(path, weights_only=False)
        exp, mll, K = blob["experiment"], blob["max_label_length"], blob["beam_width"]
        extra = {} if exp == "vitstr" else {"dec_depth": blob["dec_depth"]}
        cfg = make_config_long(exp, mll, blob["n_extra"], **extra)
        m = create_model(exp, charset_train=charset(blob["n_extra"]), max_label_length=mll, **extra)
        (m if exp == "vitstr" else m.model).load_state_dict(golden_state_dict(cfg, blob["weight_seed"], blob["sharp"]))
        m = m.eval().to("cuda")
        x = synth_images(cfg, blob["batch"], blob["image_seed"]).cuda()
        lex = m.compile_lexicon(blob["lexicon"])
        mask = m.allowlist_mask(blob["allowlist"], blob["batch"])
        with torch.inference_mode():
            ids, lengths, scores = m.model.beam_search(x, K, class_mask=mask, lexicon=lex,
                                                       roots=lex.roots_for(blob["batch"]))
        ids, lengths, scores = ids.cpu(), lengths.cpu(), scores.cpu().double()
        before = checked
        for b, im in enumerate(blob["images"]):
            g_ids, g_s = im["ids"], im["scores"]
            tg = [p + [0] for p in g_ids]
            total += len(g_ids)
            prune_ok = all(mg > TERM_MAX * (ta + tb)
                           for mg, (ta, tb) in zip(im["prune_margins"].tolist(), im["prune_terms"].tolist()))
            for k, p in enumerate(g_ids):
                n = lengths[b, k].item()
                got = ids[b, k, :n].tolist() if n >= 0 else None
                if got == p:
                    assert abs(scores[b, k].item() - g_s[k].item()) <= TERM_MAX * len(tg[k]), (blob["name"], b, k)
                gap_ok = all(abs(g_s[k].item() - g_s[j].item()) > TERM_MAX * sum(distinct_terms(tg[k], tg[j]))
                             for j in (k - 1, k + 1) if 0 <= j < len(g_ids))
                if prune_ok and gap_ok:
                    assert got == p, (blob["name"], b, k, got, p)
                    checked += 1
            if prune_ok and len(g_ids) < K:
                assert bool(torch.isneginf(scores[b, len(g_ids):]).all()) and bool((lengths[b, len(g_ids):] == -1).all())
        print(f"{blob['name']}: {checked - before} ranks checked")
    print(f"checked {checked} of {total} golden hypotheses")
    assert checked * 2 >= total, (checked, total)
