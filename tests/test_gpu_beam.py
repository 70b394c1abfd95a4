"""GPU: beam search on the device (parseq_beam_search; `PARSeq.beam_search`, `ViTSTR.beam_search`).

Beam width 1 is greedy AR decoding bit for bit: the same ids through the first EOS as `forward` on the chain of separate
kernels (ar_kernel 0, no refinement), and a score equal to the sum of log_softmax of that forward's logits.  Every
hypothesis's score agrees with the engine's own `score()` of its label; on a 3-character charset with 2-character labels,
where a beam of 16 holds every prefix and is exact, the hypotheses are the 16 best of all readings by `score()`.  An
image's hypotheses and score bits do not depend on its batch-mates, its place, the batch size, the group split or the
input format.  Allowlists constrain every expansion; a NaN crop stays in its own row."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# DESIGN section 5: engine logits within 2e-2 of the fp32 reference; a term logit - LSE moves by at most twice the largest
# logit change (tests/test_gpu_score.py).  Beam search reads the AR chain's logits (the fused LayerNorm + head kernel at
# <= 128 classes), score() the head GEMM with its log-sum-exp epilogue: both within the logit bound of the same decoder
# output, so one score differs from the other by at most TERM_MAX per term, n + 1 terms.
TERM_MAX = 2 * 2.0e-2
# log_softmax of the same fp32 logits row: only the fp32 rounding of the log-sum-exp differs (tests/test_gpu_score.py)
LSE_REL = 1.0e-5


def _model(experiment, mll=25, seed=0, n_extra=0, dec_depth=1, sharp=0.0, charset_train=None, **kw):
    from make_golden_long import charset, make_config_long
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    extra = {} if experiment == "vitstr" else {"dec_depth": dec_depth}
    cs = charset_train or charset(n_extra)
    cfg = (make_config(experiment, charset_train=cs, max_label_length=mll, **extra) if charset_train
           else make_config_long(experiment, mll, n_extra, **extra))
    sd = init_state_dict(cfg, seed, sharp=sharp)
    m = create_model(experiment, charset_train=cs, charset_test=cs, max_label_length=mll, **extra, **kw)
    (m if experiment == "vitstr" else m.model).load_state_dict(sd)
    return cfg, m.eval().to("cuda")


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _greedy(m, experiment, x, mll, mask):
    with torch.inference_mode():
        if experiment == "vitstr":
            return m.model.forward_tokens(x, None, return_ids=True, class_mask=mask)
        return m.model.forward(m.tokenizer, x, mll, return_ids=True, class_mask=mask)


# ---------------------------------------------------------------- K = 1 is greedy decoding
K1_CASES = [("parseq", 25, 0, 1), ("parseq-tiny", 25, 2906, 1), ("parseq-tiny", 25, 16289, 1), ("parseq", 25, 0, 2),
            ("parseq", 63, 0, 1), ("vitstr", 25, 0, 1)]


@pytest.mark.parametrize("allow", [False, True], ids=["free", "allowlist"])
@pytest.mark.parametrize("case", K1_CASES, ids=lambda c: f"{c[0]}-L{c[1] + 1}-C{95 + c[2]}-depth{c[3]}")
def test_width_one_is_greedy_bit_for_bit(case, allow):
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    experiment, mll, n_extra, depth = case
    kw = {} if experiment == "vitstr" else {"refine_iters": 0}
    cfg, m = _model(experiment, mll, seed=21, n_extra=n_extra, dec_depth=depth, sharp=3.0, **kw)
    if experiment != "vitstr":
        m.model.set_engine_option("ar_kernel", 0)
    N = 6
    x = synth_images(cfg, N, 22).cuda()
    cs = charset(n_extra)
    allowlist = [cs[:10], None, "abc", cs[5:40], "", cs[::3]] if allow else None
    mask = m.allowlist_mask(allowlist, N)
    logits, ids = _greedy(m, experiment, x, mll, mask)
    with torch.inference_mode():
        bids, blen, bsc = m.model.beam_search(x, 1, None, class_mask=mask)
    S = logits.shape[1]
    assert bids.shape == (N, 1, S)
    lp = torch.log_softmax(logits, -1)
    lse = torch.logsumexp(logits, -1)
    for b in range(N):
        row = ids[b].tolist()
        n = row.index(0) if 0 in row else S
        assert blen[b, 0].item() == n, b
        assert bids[b, 0, :n].tolist() == row[:n], b
        assert bool((bids[b, 0, n:] == 0).all())
        t = n + 1 if n < S else n
        ref = lp[b, :t].gather(1, ids[b, :t, None].long())[:, 0]
        bound = (LSE_REL * (1 + lse[b, :t].abs())).sum().item() + 1e-6 * t
        assert abs(bsc[b, 0].item() - ref.sum().item()) <= bound, (b, bsc[b, 0].item(), ref.sum().item())


# ---------------------------------------------------------------- against score() of the same labels
@pytest.mark.parametrize("case", [("parseq", 0, 1), ("parseq-tiny", 2906, 1), ("parseq", 0, 2), ("vitstr", 0, 1)],
                         ids=lambda c: f"{c[0]}-C{95 + c[1]}-depth{c[2]}")
def test_hypothesis_scores_equal_score_of_their_labels(case):
    from parseq_b200.weights import synth_images
    experiment, n_extra, depth = case
    cfg, m = _model(experiment, 25, seed=31, n_extra=n_extra, dec_depth=depth, sharp=2.0)
    x = synth_images(cfg, 5, 32).cuda()
    K, S = 8, 11                                   # max_length 10: 11 positions
    with torch.inference_mode():
        labels, scores = m.beam_search(x, K, max_length=S - 1)
    assert scores.shape == (5, K)
    checked = 0
    for b in range(5):
        hyp = labels[b]
        assert 1 <= len(hyp) <= K and len(set(hyp)) == len(hyp) and all(len(h) <= S for h in hyp)
        s = scores[b, :len(hyp)]
        assert bool(torch.isneginf(scores[b, len(hyp):]).all())
        assert bool((s[:-1] >= s[1:]).all()), s                  # best first
        with torch.inference_mode():
            _, terms = m.score(x[b:b + 1], hyp, return_token_logprobs=True)
        for k, h in enumerate(hyp):
            # a reading that ended with EOS: all n + 1 terms; one that filled the S positions: its S character terms
            t = len(h) + 1 if len(h) < S else len(h)
            ref = terms[0, k, :t].double().sum().item()
            assert abs(s[k].item() - ref) <= TERM_MAX * t, (b, h, s[k].item(), ref)
            checked += 1
    assert checked >= 5 * K // 2


def test_tiny_charset_beam_is_the_top16_of_every_reading():
    """3 characters and 3 positions (max_length 2): 40 readings, and a beam of 16 holds every prefix up to the last step,
    so it is exact.  Every reading is scored by the engine's own score() of a model with max_label_length 3, whose
    per-position terms 0..2 are the same AR steps: n + 1 terms for a reading that ends with EOS, 3 for one of 3
    characters.  The 16 best readings by that score are the hypotheses, rank by rank wherever the gaps to the
    neighbouring ranks exceed both scores' bounds; a reading above the 17th by more than both bounds is among them.
    Terms of a common target prefix are the same numbers in both readings, in the beam (one parent score) as in score()
    (the same causal rows), so a gap only has to exceed TERM_MAX times the terms the two readings do not share.  The
    weights carry the seeded head bias of the reference goldens (make_golden_beam.golden_state_dict), which spreads
    the readings as a trained head does."""
    import itertools
    from make_golden_beam import distinct_terms, golden_state_dict
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", 3, seed=41, sharp=4.0, charset_train="abc")
    m.model.load_state_dict(golden_state_dict(cfg, 41, 4.0))
    N = 16
    x = synth_images(cfg, N, 42).cuda()
    words = ["".join(p) for n in range(4) for p in itertools.product("abc", repeat=n)]
    with torch.inference_mode():
        labels, scores = m.beam_search(x, 16, max_length=2)
        _, terms = m.score(x, words, return_token_logprobs=True)
    checked = 0
    for b in range(N):
        full = {w: terms[b, i, :min(len(w) + 1, 3)].double().sum().item() for i, w in enumerate(words)}
        nt = {w: min(len(w) + 1, 3) for w in words}
        tg = {w: [ord(ch) for ch in w] + ([0] if len(w) < 3 else []) for w in words}

        def bound(u, w):
            return TERM_MAX * sum(distinct_terms(tg[u], tg[w]))
        assert len(labels[b]) == 16
        order = sorted(full.items(), key=lambda kv: -kv[1])
        for k, h in enumerate(labels[b]):
            assert abs(scores[b, k].item() - full[h]) <= TERM_MAX * nt[h], (b, h)
        w17, v17 = order[16]
        for w, v in order[:16]:
            if v - v17 > bound(w, w17):
                assert w in labels[b], (b, w)
        for k in range(16):
            w, v = order[k]
            if all(abs(v - order[j][1]) > bound(w, order[j][0]) for j in (k - 1, k + 1) if j >= 0):
                assert labels[b][k] == w, (b, k, labels[b][k], w)
                checked += 1
    print(f"ranks checked: {checked} of {16 * N}")
    assert checked * 2 >= 16 * N


# ---------------------------------------------------------------- invariance
def test_hypotheses_do_not_depend_on_the_rest_of_the_call():
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", seed=51, sharp=2.0)
    m.model.set_engine_option("fuse_ln", 0)          # one encoder kernel regime at every batch size
    x = synth_images(cfg, 300, 52).cuda()
    with torch.inference_mode():
        ref = m.model.beam_search(x[:1], 5)
        for N, pos in ((7, 3), (300, 0), (300, 299), (300, 130)):
            xs = x[:N].clone()
            xs[pos] = x[0]
            out = m.model.beam_search(xs, 5)
            for r, o in zip(ref, out):
                assert _same(o[pos], r[0]), (N, pos)
        m.model.set_engine_option("dec_chunk", 32)   # another group split: 6 images per group instead of 25
        out = m.model.beam_search(x[:40], 5)
        full = m.model.beam_search(x[:1], 5)
    for r, o, f in zip(ref, out, full):
        assert _same(o[0], r[0]) and _same(f[0], r[0])
    # float, uint8 and crop inputs
    rng = np.random.default_rng(53)
    u8 = torch.from_numpy(rng.integers(0, 256, (3, 32, 128, 3), dtype=np.uint8))
    xf = ((u8.permute(0, 3, 1, 2).to(torch.float32).div(255) - 0.5) / 0.5).cuda()
    crops = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).cuda() for h, w in ((20, 70), (64, 300), (32, 128))]
    with torch.inference_mode():
        a = m.model.beam_search(xf, 4)
        b = m.model.beam_search(u8.cuda(), 4)
        for p, q in zip(a, b):
            assert _same(p, q)
        c = m.beam_search(crops, 4, rotation=90)
        d = m.beam_search(m.preprocess(crops, 90), 4)
        e = m.beam_search([cr.cpu() for cr in crops], 4, rotation=90)
    assert c[0] == d[0] == e[0] and _same(c[1], d[1])
    assert e[1].device.type == "cpu" and _same(e[1], d[1].cpu())


def test_vitstr_hypotheses_do_not_depend_on_the_batch():
    from parseq_b200.weights import synth_images
    cfg, m = _model("vitstr", seed=55, sharp=2.0)
    x = synth_images(cfg, 70, 56).cuda()
    with torch.inference_mode():
        ref = m.model.beam_search(x[:1], 6)
        xs = x.clone()
        xs[69] = x[0]
        out = m.model.beam_search(xs, 6)
    for r, o in zip(ref, out):
        assert _same(o[69], r[0])


# ---------------------------------------------------------------- allowlists, non-finite crops, memory
@pytest.mark.parametrize("experiment", ["parseq", "vitstr"])
def test_allowlists_constrain_every_hypothesis(experiment):
    from parseq_b200.weights import synth_images
    cfg, m = _model(experiment, seed=61, sharp=2.0)
    x = synth_images(cfg, 4, 62).cuda()
    allow = ["0123456789", "", None, "xyz"]
    with torch.inference_mode():
        labels, scores = m.beam_search(x, 6, allowlist=allow)
        ids, lengths, raw = m.model.beam_search(x, 6, class_mask=m.allowlist_mask(allow, 4))
    for b, a in enumerate(allow):
        if a is not None:
            assert all(set(h) <= set(a) for h in labels[b]), (b, labels[b])
    assert labels[1] == [""] and scores[1, 0].item() == 0.0
    assert bool(torch.isneginf(scores[1, 1:]).all()) and lengths[1, 1:].tolist() == [-1] * 5
    assert len(labels[3]) == 6 and len(labels[2]) == 6


@pytest.mark.parametrize("experiment", ["parseq", "vitstr"])
def test_nan_crop_stays_in_its_own_row(experiment):
    from parseq_b200.weights import synth_images
    cfg, m = _model(experiment, seed=71)
    x = synth_images(cfg, 5, 72).cuda()
    with torch.inference_mode():
        ref = m.model.beam_search(x, 4)
        xn = x.clone()
        xn[2] = float("nan")
        out = m.model.beam_search(xn, 4)
    keep = torch.tensor([0, 1, 3, 4], device="cuda")
    for r, o in zip(ref, out):
        assert _same(o[keep], r[keep])


def test_no_beam_buffers_until_the_first_beam_call_and_forward_unchanged():
    from parseq_b200.weights import synth_images
    cfg, m = _model("parseq", seed=81)
    x = synth_images(cfg, 16, 82).cuda()
    with torch.inference_mode():
        a = m(x)
        eng = m.model.engine()
        assert eng.debug_int("beam_bytes") == 0
        m.score(x, ["abc"])
        assert eng.debug_int("beam_bytes") == 0
        eng.set_option("timing", 1)
        m.beam_search(x, 3)
        torch.cuda.synchronize()
        t = eng.get_timing()
        eng.set_option("timing", 0)
        assert eng.debug_int("beam_bytes") > 0
        assert t["beam_select"]["launches"] >= cfg.max_label_length + 1
        b = m(x)
    assert _same(a, b)


# ---------------------------------------------------------------- against the reference goldens (tests/make_golden_beam.py)
def test_beams_match_reference_goldens():
    """The fp64 beams of the reference's own modules (tests/make_golden_beam.py).  Every engine hypothesis equal to the
    golden's at its rank has a score within TERM_MAX per term of the golden's.  Where fp32 rounding cannot reorder
    anything, the labels match rank by rank: every pruning margin of the image, and the gaps to the neighbouring final
    ranks, exceed TERM_MAX times the number of terms the two scores do not share (terms of a common target prefix are
    the same numbers in both: the engine carries one parent score to all its children).  The filter keeps at least
    half of all golden hypotheses, so the test cannot pass vacuously."""
    import glob
    import os
    from make_golden_beam import distinct_terms, golden_state_dict
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import synth_images
    paths = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "beam", "bm_*.pt")))
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
        L = mll + 1
        mask = m.allowlist_mask(blob["allowlist"], blob["batch"])
        with torch.inference_mode():
            ids, lengths, scores = m.model.beam_search(x, K, class_mask=mask)
        ids, lengths, scores = ids.cpu(), lengths.cpu(), scores.cpu().double()
        before = checked
        for b, im in enumerate(blob["images"]):
            g_ids, g_s = im["ids"], im["scores"]
            tg = [p + [0] if len(p) < L else p for p in g_ids]          # target sequences: characters, then EOS
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
