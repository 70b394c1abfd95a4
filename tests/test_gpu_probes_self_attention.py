"""GPU: the decoder self-attention on the probes of tests/probe_models.py, against their fp64 model, route by route.

`dec_self_order` makes the latest visible key (and, on a second head, that key's token in the image's own ids) decide
two flip pairs, and the earliest visible key a third: a causal or cloze mask off by one key, a padding mask that starts
late or hides only the EOS keys, an extra zero key, or a read of another image's ids, table rows or cache rows moves
the output by 1 or more.  `dec_self_query` makes norm_q's and norm_c's LayerNorm eps and the query's bits below bf16
decide two more.  tests/test_probe_separation_cpu.py shows every such bug 10x over the tolerance of 1e-4 in each pass
it touches, while a correct engine agrees with the fp64 model to ~1e-6.

Every probe image has its own forced ids and its own first EOS.  The probes run through every cluster-kernel
instantiation of test_gpu_decoder_isolated.py (proven by the full reach tuple; the AR loop puts the latest visible key
on both sides of every 8-key group edge of the kernel's online softmax), the grid-barrier kernel, the chain at L = 26
(one key per lane) and L = 64 (two), NAR, one and two refinement passes with the first EOS at 1, 31, 32, 33 and 63 or
absent at L = 64 (both 32-key ballot groups), depth 2 (the rows kernels over the table and over the per-image caches)
and `model.decode` with a query mask, a padding mask and, at depth 2, a content mask, each hiding a key that would win.
`score` runs them (and `dec_cross`, `dec_ln_eps`) as teacher-forced candidates at 95 and 16384 classes and depth 2.
Each case prints its error (run with -s to see it)."""
import pytest
import torch

import probe_models as pm
from test_gpu_decoder_isolated import AR_CASES as DEC_AR_CASES
from test_gpu_decoder_isolated import ROUTES as DEC_AR_ROUTES
from test_gpu_probes import _check, _engine, _probe, _repeat, _run

pytestmark = pytest.mark.gpu

KINDS = pm.SELF_KINDS


def _name(fn):
    return fn.__name__


# ---- every cluster-kernel instantiation -------------------------------------------------------------------------------
AR_CASES = [(fn, D, r, wide, pitch) for fn in KINDS for D, r, wide, pitch in DEC_AR_CASES]


def _ar_id(c):
    fn, D, (mt, cs, hs), wide, pitch = c
    return f"{_name(fn)}-D{D}-mt{mt}-cs{cs}-hs{hs}-{'wide' if wide else 'c95'}-idp{pitch}"


@pytest.mark.parametrize("case", AR_CASES, ids=[_ar_id(c) for c in AR_CASES])
def test_self_attention_probe_cluster_instantiation(case):
    fn, D, (mt, cs, hs), wide, pitch = case
    p = _probe(fn, (D, 1), None, pm.WIDE_EXTRA if wide else 0, 25 if pitch == 32 else 63)
    B, opts = DEC_AR_ROUTES[(mt, cs, hs)]
    if B is None:
        B = 2 if D == 192 else 1
    m = _engine(p)
    m.model.decode_ar, m.model.refine_iters = True, 0
    got, ref = _run(p, B, opts)
    reached = tuple(m.model.engine().debug_int(k) for k in ("ar_last_path", "ar_last_mt", "ar_last_cluster_size",
                                                            "ar_last_head_split", "ar_last_wide", "ar_last_ids_pitch"))
    assert reached == (2, mt, cs, hs, wide, pitch), reached
    _check(p, _ar_id(case), got, ref)


# ---- the other AR routes and passes -----------------------------------------------------------------------------------
# name -> (engine options, decode_ar, refine_iters, the ar_last_path reached or None)
ROUTES = {
    "grid-barrier": ((("ar_kernel", 1),), True, 0, 1),
    "chain": ((("ar_kernel", 0),), True, 0, 0),
    "nar": ((), False, 0, None),
    "refine": ((), True, 1, None),
    "refine2": ((), True, 2, None),
}
CASES = [(fn, (D, 1), mll, r) for fn in KINDS for D in (192, 384, 768) for mll in (25, 63) for r in ROUTES
         if not (r == "grid-barrier" and (mll == 63 or D == 768)) and not (r == "refine2" and D != 384)]
CASES += [(fn, (384, 2), mll, r) for fn in KINDS for mll in (25, 63) for r in ("chain", "nar", "refine")]


def _case_id(c):
    fn, key, mll, r = c
    return f"{_name(fn)}-D{key[0]}-depth{key[1]}-L{mll + 1}-{r}"


def _run_refine2(p, B):
    """Two refinement passes: the first over another context, the second over the probe's; the logits are the second's."""
    m = _engine(p)
    for k, v in (("fuse_ln", 0), ("ar_kernel", 2), ("ar_cluster_size", 0), ("ar_clusters", 0)):
        m.model.set_engine_option(k, v)
    L, C, bos = p.cfg.max_label_length + 1, p.cfg.num_classes, p.cfg.num_tokens - 2
    x = _repeat(p.images, B).cuda()
    forced = _repeat(p.forced, B)
    ctx = _repeat(p.context, B)
    first = pm.self_context(B, L, C, bos, (5, None, 2), 77)
    with torch.inference_mode():
        mem = m.model.encode(x)
        got = m.model.forward(m.tokenizer, x, p.cfg.max_label_length, forced_ids=forced,
                              forced_refine=torch.stack([first, ctx]))
    memr = mem.to(torch.bfloat16).float()
    assert torch.equal(memr.cpu(), _repeat(p.memory(), B)), "the probe's memory is not the +-1 pattern"
    q = pm.Probe(**{**p.__dict__, "images": x.cpu(), "forced": forced, "context": ctx})
    return got, q.expected(device="cuda", memory=memr, pass_="refine")


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_self_attention_probe(case):
    fn, key, mll, route = case
    p = _probe(fn, key, None, 0, mll)
    opts, ar, refine, path = ROUTES[route]
    m = _engine(p)
    m.model.decode_ar, m.model.refine_iters = ar, refine
    if refine == 2:
        got, ref = _run_refine2(p, pm.SELF_B)
    else:
        got, ref = _run(p, pm.SELF_B, opts)
    if path is not None:
        assert m.model.engine().debug_int("ar_last_path") == path
    _check(p, route, got, ref)


# ---- model.decode: caller masks (mode 2) ------------------------------------------------------------------------------
def _decode_masks(B, NQ, J):
    """Masks that each hide a key that would win if visible: the query mask hides the latest key J - 1 from the even
    queries, the padding mask hides key J - 2 of the odd images (the latest left to their even queries) and key J - 1 of
    image 2, and the content mask (causal) also hides content rows 17..19 their own key, so that the latest key those
    rows see, whose parity layer 1's head 3 reads at depth 2, is the one before."""
    qmask = torch.zeros((NQ, J), dtype=torch.bool)
    qmask[::2, J - 1] = True
    pmask = torch.zeros((B, J), dtype=torch.bool)
    pmask[1::2, J - 2] = True
    pmask[2, J - 1] = True
    cmask = torch.triu(torch.ones((J, J), dtype=torch.bool), 1)
    for k in (J - 3, J - 2, J - 1):
        cmask[k, k] = True
    return qmask, pmask, cmask


@pytest.mark.parametrize("depth", [1, 2])
def test_self_attention_probe_decode_with_masks(depth):
    """parseq_decode_ex (mode 2) on dec_self_order with the masks of _decode_masks: the latest visible key wins, so each
    mask decides the output (checked on the fp64 model: dropping any one of them moves it by 1 or more).  The content
    mask acts at depth 2 only, where head 3 of layer 1 reads what the content stream saw under it; queries are the
    probe's own position queries, so every row stays a +-1 pattern."""
    from decoder_reference import DecoderReference, DepthDecoderReference
    p = _probe(pm.dec_self_order, (384, depth))
    m = _engine(p)
    for k, v in (("fuse_ln", 0), ("ar_kernel", 2)):
        m.model.set_engine_option(k, v)
    B, J = pm.SELF_B, 20
    NQ = p.cfg.max_label_length + 1
    tgt = p.forced[:, :J].long()
    query = p.sd["pos_queries"][:, :NQ].float()
    qmask, pmask, cmask = _decode_masks(B, NQ, J)
    x = p.images.cuda()
    with torch.inference_mode():
        mem = m.model.encode(x)
        out = m.model.decode(tgt.cuda(), mem, tgt_mask=cmask.cuda(), tgt_padding_mask=pmask.cuda(),
                             tgt_query=query.cuda(), tgt_query_mask=qmask.cuda())
        got = m.model.head(out)
    memr = mem.to(torch.bfloat16).float()
    assert torch.equal(memr.cpu(), p.memory()), "the probe's memory is not the +-1 pattern"
    model = (DepthDecoderReference if depth > 1 else DecoderReference)(p.cfg, p.sd, device="cuda")
    q = query.to("cuda", torch.float64).expand(B, -1, -1)
    causal = torch.triu(torch.ones((J, J), dtype=torch.bool), 1)

    def ref_of(qm, pmk, cm):
        args = (tgt.cuda(), model._memory(memr), q, qm.cuda(), pmk.cuda())
        return model._decode(*args, cm.cuda()) if depth > 1 else model._decode(*args)

    ref = ref_of(qmask, pmask, cmask)
    assert got.shape == ref.shape == (B, NQ, p.cfg.num_classes)
    variants = {"query mask": (torch.zeros_like(qmask), pmask, cmask), "padding mask": (qmask, torch.zeros_like(pmask), cmask)}
    if depth > 1:
        variants["content mask"] = (qmask, pmask, causal)
    for what, masks in variants.items():
        assert (ref - ref_of(*masks)).abs().max() >= 1.0, f"the {what} does not decide the probe"
    _check(p, f"decode depth {depth}", got, ref)


# ---- score(): teacher-forced candidates through the scoring pass ---------------------------------------------------------
# (builder, key, extra classes): the probes' heads are class-dependent, so log_softmax sees every flip
SCORE_CASES = [(fn, (384, 1), 0) for fn in (pm.dec_self_order, pm.dec_self_query, pm.dec_cross, pm.dec_ln_eps)]
SCORE_CASES += [(fn, (384, 2), 0) for fn in (pm.dec_self_order, pm.dec_self_query, pm.dec_cross)]
SCORE_CASES += [(fn, (192, 1), 16384 - 95) for fn in (pm.dec_self_order, pm.dec_cross)]
PER_IMAGE = (3, 70, 1, 5, 2, 9, 4)       # image 1 has more than 64 candidate rows


def _candidates(cfg, seed):
    """targets [M, L] (c_1..c_n, EOS, 0...) of lengths 1..max_label_length, image-major, PER_IMAGE per image."""
    g = torch.Generator().manual_seed(seed)
    L, C = cfg.max_label_length + 1, cfg.num_classes
    M = sum(PER_IMAGE)
    lengths = torch.randint(1, L, (M,), generator=g, dtype=torch.int32)
    lengths[:3] = torch.tensor([1, L - 1, 2], dtype=torch.int32)
    targets = torch.randint(1, C, (M, L), generator=g, dtype=torch.int32)
    for i in range(M):
        targets[i, lengths[i]:] = 0
    return targets, lengths


@pytest.mark.parametrize("case", SCORE_CASES, ids=[f"{_name(c[0])}-D{c[1][0]}-depth{c[1][1]}-C{95 + c[2]}"
                                                   for c in SCORE_CASES])
def test_probe_through_score(case):
    """`score` with token terms against fp64 log_softmax of the probe's teacher-forced logits, candidate by candidate:
    lengths from 1 to max_label_length in one call (rows sit in groups longer than their own label), and one image
    with 70 candidates (the grouped cross kernel spans grid.y >= 2)."""
    fn, key, extra = case
    p = _probe(fn, key, None, extra)
    m = _engine(p)
    for k, v in (("fuse_ln", 0), ("ar_kernel", 2)):
        m.model.set_engine_option(k, v)
    N = len(PER_IMAGE)
    targets, lengths = _candidates(p.cfg, 50 + key[1])
    M = targets.shape[0]
    x = _repeat(p.images, N).cuda()
    with torch.inference_mode():
        scores, terms = m.model.score(x, targets, lengths, torch.tensor(PER_IMAGE, dtype=torch.int32),
                                      return_token_logprobs=True)
    forced = torch.cat([torch.full((M, 1), p.cfg.num_tokens - 2, dtype=torch.int32), targets[:, :-1]], dim=1)
    mem = p.memory()[:1].expand(M, -1, -1)
    q = pm.Probe(**{**p.__dict__, "forced": forced})
    ref = q.score_terms(device="cuda", memory=mem.cuda())
    _check(p, "score terms", terms, ref)
    # the score is an fp32 sum of up to L terms: on top of the terms' tolerance, one fp32 rounding of |score| per term
    total = ref.sum(1)
    e = (scores.double() - total).abs()
    bound = p.tol + q.cfg.max_label_length * 2.0 ** -24 * total.abs()
    print(f"[{p.name} score] max |engine - model| {e.max().item():.2e}  largest |score| {total.abs().max().item():.1f}")
    assert torch.isfinite(scores).all() and bool((e <= bound).all()), (p.name, e.max().item())
