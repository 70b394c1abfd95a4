"""GPU: candidate scoring (parseq_score; `PARSeq.score`, `lexicon_decode`, `ViTSTR.score`).

Checked against the fp64 goldens of the reference's own modules (tests/golden/score), against the engine's own module API
on the same memory (only the fp32 log-sum-exp rounding may differ), against greedy decoding, and for the properties that
need no reference: a candidate's bits do not depend on the other candidates, their number or order, the image's place in
the batch or the batch size; float, uint8 and crop inputs agree bit for bit; the encoder runs once per image; a NaN crop
stays in its own scores.  Fed the engine's own memory, the per-position terms stay within the decoder's error budget
(tests/score_budget.py) of the fp64 rounding-point model, which injected mask and query-position bugs exceed."""
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "score")
CASES = sorted(glob.glob(os.path.join(GOLDEN, "sc_*.pt")))
# DESIGN section 5: engine logits within 2e-2 (max) and 3e-3 (mean) of the fp32 reference.  A term is
# logit[t] - logsumexp(row): its error is at most the target logit's error plus the largest logit error of the row
# (logsumexp moves by at most max |d logit|), so 2x the logit bounds per term, and n + 1 of them per score.
TERM_MAX = 2 * 2.0e-2
TERM_MEAN = 2 * 3.0e-3
# The tail against log_softmax of the engine's own fp32 logits: the logits are the same bits (same GEMM, same rows), the
# log-sum-exp is merged from 128-column partials instead of torch's reduction order: fp32 rounding of the sum of
# exponentials (relative ~1e-7 per add, ~1e-6 over 16384 classes) and of log / subtraction, a few ulps of the row's
# log-sum-exp.  Bound per term: 1e-5 relative to (1 + |log-sum-exp|).
LSE_REL = 1.0e-5


def _model(experiment, mll=25, seed=0, n_extra=0, dec_depth=1, sharp=0.0, **kw):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    extra = {} if experiment == "vitstr" else {"dec_depth": dec_depth}
    cfg = make_config_long(experiment, mll, n_extra, **extra)
    sd = init_state_dict(cfg, seed, sharp=sharp)
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=mll, **extra, **kw)
    (m if experiment == "vitstr" else m.model).load_state_dict(sd)
    return cfg, sd, m.eval().to("cuda")


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _words(cs, seed, k, lo=3, hi=12):
    r = np.random.default_rng(seed)
    return ["".join(cs[i] for i in r.integers(0, len(cs), r.integers(lo, hi + 1))) for _ in range(k)]


# ---------------------------------------------------------------- against the reference goldens
@pytest.mark.parametrize("path", CASES, ids=lambda p: os.path.basename(p)[:-3])
def test_scores_match_reference_goldens(path):
    from parseq_b200.weights import synth_images
    blob = torch.load(path, weights_only=False)
    cfg, sd, m = _model(blob["experiment"], blob["max_label_length"], blob["weight_seed"], blob["n_extra"],
                        blob["dec_depth"], blob["sharp"])
    x = synth_images(cfg, blob["batch"], blob["image_seed"]).cuda()
    with torch.inference_mode():
        s, t = m.score(x, blob["candidates"], return_token_logprobs=True)
    per = [len(r) for r in blob["candidates"]]
    rows = torch.cat([s[b, :k] for b, k in enumerate(per)]).double().cpu()
    terms = torch.cat([t[b, :k] for b, k in enumerate(per)]).double().cpu()
    n = torch.tensor([len(c) for r in blob["candidates"] for c in r])
    valid = torch.arange(terms.shape[1])[None, :] <= n[:, None]
    err = (terms - blob["terms"]).abs()
    print(f"{blob['name']}: term err max {err[valid].max().item():.2e} mean {err[valid].mean().item():.2e}")
    assert bool((terms[~valid] == 0).all())
    assert err[valid].max().item() <= TERM_MAX and err[valid].mean().item() <= TERM_MEAN
    assert bool(((rows - blob["scores"]).abs() <= TERM_MAX * (n + 1)).all())
    for b, k in enumerate(per):
        assert bool(torch.isneginf(s[b, k:]).all())
    # lexicon decoding picks the golden's best candidate wherever its margin exceeds both scores' bounds
    labels, best = m.lexicon_decode(x, blob["candidates"])
    o = 0
    for b, row in enumerate(blob["candidates"]):
        g = blob["scores"][o:o + len(row)]
        top = int(g.argmax())
        ok = all(g[top] - g[j] > TERM_MAX * (len(row[top]) + len(row[j]) + 2) for j in range(len(row)) if j != top)
        if ok:
            assert labels[b] == row[top], (b, labels[b], row[top])
        assert best[b].item() == s[b].max().item()
        o += len(row)


# ---------------------------------------------------------------- the tail against the engine's own module API
@pytest.mark.parametrize("n_extra", [0, 2906, 16289], ids=["C95", "C3001", "C16384"])
def test_tail_equals_log_softmax_of_the_module_api(n_extra):
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny" if n_extra else "parseq", n_extra=n_extra, seed=5)
    cs = charset(n_extra)
    B = 3
    x = synth_images(cfg, B, 6).cuda()
    cands = [_words(cs, 10 + b, 4, 0, 25) + [""] for b in range(B)]
    with torch.inference_mode():
        s, t = m.score(x, cands, return_token_logprobs=True)
        mem = m.model.encode(x)
        tok = m.tokenizer
        flat = [(b, c) for b, r in enumerate(cands) for c in r]
        P = max(len(c) for _, c in flat) + 1
        tgt = torch.full((len(flat), P + 1), tok.pad_id, dtype=torch.long)
        for i, (_, c) in enumerate(flat):
            ids = [tok.bos_id] + tok._tok2ids(c) + [tok.eos_id]
            tgt[i, :len(ids)] = torch.tensor(ids)
        causal = torch.triu(torch.ones((P, P), dtype=torch.bool), 1).cuda()
        memory = mem[torch.tensor([b for b, _ in flat])].contiguous()
        out = m.model.decode(tgt[:, :-1].cuda(), memory, causal, None, None, causal)
        logits = m.model.head(out)
        lp = torch.log_softmax(logits, -1)
        lse = torch.logsumexp(logits, -1)
    for i, (b, c) in enumerate(flat):
        k = cands[b].index(c)
        n = len(c)
        ref = lp[i, :n + 1].gather(1, tgt[i, 1:n + 2].cuda()[:, None])[:, 0]
        bound = LSE_REL * (1 + lse[i, :n + 1].abs())
        assert bool(((t[b, k, :n + 1] - ref).abs() <= bound).all()), (i, (t[b, k, :n + 1] - ref).abs().max().item())
        assert abs(s[b, k].item() - ref.sum().item()) <= bound.sum().item() + 1e-6 * (n + 1)


def test_vitstr_tail_equals_log_softmax_of_forward_tokens():
    from parseq_b200.weights import synth_images
    from make_golden_long import charset
    cfg, sd, m = _model("vitstr", seed=7)
    x = synth_images(cfg, 4, 8).cuda()
    cands = _words(charset(0), 11, 6, 0, 25)
    with torch.inference_mode():
        s, t = m.score(x, cands, return_token_logprobs=True)
        logits = m.model.forward_tokens(x, None)
    lp = torch.log_softmax(logits, -1)
    lse = torch.logsumexp(logits, -1)
    tok = m.tokenizer
    for b in range(4):
        for k, c in enumerate(cands):
            n = len(c)
            ids = torch.tensor(tok._tok2ids(c) + [0], device="cuda")
            ref = lp[b, :n + 1].gather(1, ids[:, None])[:, 0]
            # the target logit is a dot product over D in fp32 (not the GEMM's accumulation order): a few ulps more
            bound = LSE_REL * (1 + lse[b, :n + 1].abs() + logits[b, :n + 1].abs().amax(-1))
            assert bool(((t[b, k, :n + 1] - ref).abs() <= bound).all())


# ---------------------------------------------------------------- consistency with greedy decoding
def test_score_of_the_greedy_label_is_its_log_confidence():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", seed=3, sharp=4.0, refine_iters=0)
    m.model.set_engine_option("ar_kernel", 0)
    x = synth_images(cfg, 8, 9).cuda()
    with torch.inference_mode():
        logits = m.model.forward(m.tokenizer, x, cfg.max_label_length)
        labels, conf = m.postprocess(logits)
        keep = [b for b, lb in enumerate(labels) if len(lb) <= cfg.max_label_length]   # an EOS was decoded
        assert keep
        s = m.score(x[keep], [[labels[b]] for b in keep])
    for i, b in enumerate(keep):
        lb = labels[b]
        # the chain's AR steps take the fused LayerNorm + head kernel, the score the head GEMM: logit bounds per term
        assert abs(s[i, 0].item() - float(np.log(conf[b]))) <= TERM_MAX * (len(lb) + 1), (b, lb, s[i, 0].item(), conf[b])


# ---------------------------------------------------------------- invariance
def test_score_bits_do_not_depend_on_the_rest_of_the_call():
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", seed=4)
    m.model.set_engine_option("fuse_ln", 0)          # one encoder kernel regime at every batch size
    cs = charset(0)
    probe = ["", "a", "hello", "0123456789abcdefghijklmno"]
    x = synth_images(cfg, 1030, 12).cuda()
    lex = _words(cs, 13, 996, 1, 25)
    with torch.inference_mode():
        ref = m.score(x[:1], probe)[0]
        # other candidates, their number (K = 1 .. 1000) and order
        for k in range(len(probe)):
            assert _same(m.score(x[:1], [probe[k]])[0, 0], ref[k])
        big = probe[::-1] + lex
        s = m.score(x[:1], big)[0]
        assert _same(s[:4].flip(0), ref)
        # the image's position in the batch and the batch size, super-chunks included (max_batch = 512)
        for N, pos in ((7, 5), (512, 300), (1030, 1029), (1030, 600)):
            xs = x[:N].clone()
            xs[pos] = x[0]
            cands = [["zz", "q"]] * N
            cands[pos] = probe
            s = m.score(xs, cands)
            assert _same(s[pos, :4], ref), N
    # float, uint8 and crop inputs
    rng = np.random.default_rng(14)
    u8 = torch.from_numpy(rng.integers(0, 256, (3, 32, 128, 3), dtype=np.uint8))
    xf = ((u8.permute(0, 3, 1, 2).to(torch.float32).div(255) - 0.5) / 0.5).cuda()   # on the CPU: IEEE division, as torchvision
    u8 = u8.cuda()
    crops = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).cuda() for h, w in ((20, 70), (64, 300), (32, 128))]
    with torch.inference_mode():
        a = m.score(xf, probe)
        b = m.score(u8, probe)
        assert _same(a, b)
        c = m.score(crops, probe, rotation=90)
        d = m.score(m.preprocess(crops, 90), probe)
        assert _same(c, d)
        e = m.score([cr.cpu() for cr in crops], probe, rotation=90)
        assert e.device.type == "cpu" and _same(e, d.cpu())


def test_forward_bits_unchanged_by_a_score_call():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", seed=2)
    x = synth_images(cfg, 16, 15).cuda()
    with torch.inference_mode():
        a = m(x)
        m.score(x, ["abc", "hello", ""])
        b = m(x)
    assert _same(a, b)


def test_encoder_runs_once_per_image():
    from parseq_b200.weights import synth_images
    from make_golden_long import charset
    cfg, sd, m = _model("parseq", seed=6)
    x = synth_images(cfg, 20, 16).cuda()
    eng = m.model.engine()
    counts = {}
    for K in (1, 50):
        eng.set_option("timing", 0)
        eng.set_option("timing", 1)
        with torch.inference_mode():
            m.score(x, _words(charset(0), 17, K, 1, 25))
        torch.cuda.synchronize()
        counts[K] = eng.get_timing()
        eng.set_option("timing", 0)
    assert counts[1]["enc_gemm"]["launches"] == counts[50]["enc_gemm"]["launches"] > 0
    assert counts[50]["score_tail"]["launches"] > 0


def test_nan_crop_gives_nan_for_its_own_scores_only():
    from parseq_b200.weights import synth_images
    from make_golden_long import charset
    for exp in ("parseq", "vitstr"):
        cfg, sd, m = _model(exp, seed=8)
        x = synth_images(cfg, 5, 18).cuda()
        lex = _words(charset(0), 19, 7, 0, 25)
        with torch.inference_mode():
            ref = m.score(x, lex)
            xn = x.clone()
            xn[2] = float("nan")
            s = m.score(xn, lex)
        assert bool(torch.isnan(s[2]).all()), exp
        keep = torch.tensor([0, 1, 3, 4])
        assert _same(s[keep], ref[keep]), exp


# ---------------------------------------------------------------- decoder budget of the scoring pass
@pytest.mark.parametrize("key", [(192, 1), (384, 1), (384, 2)], ids=lambda k: f"D{k[0]}-depth{k[1]}")
def test_scoring_pass_within_the_decoder_budget(key):
    """Fed the engine's own memory (fuse_ln = 0: `encode` returns the fp32 LayerNorm output whose bf16 copy the decoder
    reads, in the regime the score call runs), the per-position terms stay within tests/score_budget.py's bounds of the
    fp64 rounding-point model of tests/decoder_reference.py (twice the decoder's logit bounds, reason stated there and
    shown by tests/test_score_budget_cpu.py), while the model with the self_mask_leak or pos_query_shift bug - a causal
    mask that lets position i see key i + 1, an off-by-one query position - lies 2x or more outside them."""
    from decoder_reference import DecoderReference, DepthDecoderReference
    from make_golden_long import charset
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict, synth_images
    from score_budget import SCORE_BUGS, forcing, model_terms, term_excess, term_stats, words
    D, depth = key
    exp = {192: "parseq-tiny", 384: "parseq"}[D]
    over = dict(enc_depth=2, charset_train=charset(0), max_label_length=25, dec_depth=depth)
    cfg = make_config(exp, **over)
    sd = init_state_dict(cfg, 21, sharp=4.0)
    m = create_model(exp, **over)
    m.model.load_state_dict(sd)
    m = m.eval().to("cuda")
    m.model.set_engine_option("fuse_ln", 0)
    B, K = 6, 4
    x = synth_images(cfg, B, 61).cuda()
    cands = [words(cfg.charset_train, 30 + b, K, cfg.max_label_length) for b in range(B)]
    with torch.inference_mode():
        _, t = m.score(x, cands, return_token_logprobs=True)
        mem = m.model.encode(x)
    flat = [c for r in cands for c in r]
    img = torch.arange(B).repeat_interleave(K).cuda()
    ids, tgt, valid = forcing(m.tokenizer, flat, cfg.max_label_length + 1)
    got = t.reshape(B * K, -1)
    model = DepthDecoderReference if depth > 1 else DecoderReference
    ref_logits = model(cfg, sd, device="cuda").ar(mem[img], ids)
    ref = model_terms(ref_logits, tgt, valid)
    s = term_stats(got, ref, ref_logits, valid)
    print(f"engine D{D} depth {depth}: {s}")
    assert max(term_excess(s, key).values()) <= 1.0, s
    for bug in SCORE_BUGS:
        bad = model_terms(model(cfg, sd, device="cuda", bug=bug).ar(mem[img], ids), tgt, valid)
        sb = term_stats(got, bad, ref_logits, valid)
        print(f"  vs {bug}: {sb}")
        assert max(term_excess(sb, key).values()) >= 2.0, (bug, sb)
