"""GPU: character maps for given text - the cross-attention maps of scored candidates (parseq_score_args.attn_maps) and
of beam hypotheses (parseq_beam_args.attn_maps, plain and under a lexicon), and locate(text=).

  * Identity: a candidate equal to the greedy AR reading (no refinement) gets read_with_attention's maps, bit for bit;
    a beam hypothesis gets the score maps of its label, bit for bit (at K = 1 the AR maps); the lexicon beam's word gets
    the score maps of that word.
  * Invariance: an image's maps are bitwise the same whatever the candidate counts of its neighbours (1, 10, 100), the
    group and super-chunk splits (dec_chunk, max_batch < N) and the input form (raw crops, their uint8 stack).
  * Nothing else changes: scores, token terms, beam ids, lengths and scores are bit-identical with and without maps.
  * Accuracy: against the maps of the reference's own fp64 modules (tests/golden/alignment) within GOLDEN_BOUNDS, and
    against the fp64 rounding-point maps of tests/attn_maps_reference.py fed the engine's bf16 memory and the
    candidates' ids, within its BOUNDS, at C = 95 / 3001 / 16384, depth 1 and 2, L = 26 and 64, T = 32 / 65 / 130 /
    256.
  * The cross-attention probe of tests/probe_models.py drives the grouped maps kernel at T = 32, 65, 130, 240 and
    256, next to a seeded image, to 1e-4 of the fp64 maps.
  * The live-bytes and live-object counts return to their start after calls with maps; locate(text=) of the greedy
    reading places every character where locate does, also on rotated crops."""
import functools
import gc
import os

import pytest
import torch

from attn_maps_reference import BOUNDS, GOLDEN_BOUNDS, MapsReference, excess, format_stats, map_stats
from token_count_geometries import geometry_config

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=8)
def _model(exp="parseq", T=None, mll=25, depth=1, n_extra=0):
    from make_golden_long import charset
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from make_golden_attention import golden_state_dict
    over = dict(geometry_config(T, exp)[1]) if T is not None else dict(enc_depth=2)
    over.update(max_label_length=mll, dec_depth=depth, charset_train=charset(n_extra))
    cfg = make_config(exp, **over)
    sd = golden_state_dict(cfg, 5, 4.0)             # sharp attention, a seeded head bias: most readings end early
    m = create_model(exp, **over)
    m.model.load_state_dict(sd)
    m = m.eval().to("cuda")
    m.model.set_engine_option("fuse_ln", 0)         # encode() returns the memory the decoder reads
    m.model.decode_ar, m.model.refine_iters = True, 0
    return cfg, sd, m


def _images(cfg, B, seed):
    from parseq_b200.weights import synth_images
    return synth_images(cfg, B, seed).cuda()


def _words(cfg, n, seed, max_len=None):
    g = torch.Generator().manual_seed(seed)
    cs = cfg.charset_train
    top = cfg.max_label_length if max_len is None else max_len
    out = []
    for _ in range(n):
        k = int(torch.randint(0, top + 1, (1,), generator=g))
        out.append("".join(cs[int(i)] for i in torch.randint(0, len(cs), (k,), generator=g)))
    return out


def _score(m, x, cands, **kw):
    with torch.inference_mode():
        return m.score(x, cands, return_token_logprobs=True, return_attention=True, **kw)


def _flat(maps):
    return maps.reshape(*maps.shape[:-2], -1)


# ---- identity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [(None, 25, 1, 0), (None, 25, 2, 0), (None, 63, 1, 0), (None, 25, 1, 2906), (130, 25, 1, 0)],
                         ids=["s", "d2", "l64", "c3001", "t130"])
def test_score_maps_of_the_greedy_reading_are_read_with_attention(case):
    T, mll, depth, n_extra = case
    cfg, _, m = _model("parseq", T, mll, depth, n_extra)
    x = _images(cfg, 7, 11)
    with torch.inference_mode():
        logits, read = m.read_with_attention(x)
    labels, _ = m.postprocess(logits)
    ended = [b for b, lab in enumerate(labels) if len(lab) <= mll]     # a reading without EOS is no label to score
    assert len(ended) >= 4, labels
    _, _, maps = _score(m, x[ended], [[labels[b]] for b in ended])
    for j, b in enumerate(ended):
        n = len(labels[b])
        assert torch.equal(maps[j, 0, :n + 1], read[b, :n + 1]), (b, labels[b])
        assert not bool(maps[j, 0, n + 1:].any())


@pytest.mark.parametrize("case", [(1, 25, 1, 0), (4, 25, 1, 0), (5, 25, 2, 0), (3, 63, 1, 0), (4, 25, 1, 2906)],
                         ids=["k1", "k4", "k5-d2", "k3-l64", "k4-c3001"])
def test_beam_maps_are_the_score_maps_of_each_hypothesis(case):
    K, mll, depth, n_extra = case
    cfg, _, m = _model("parseq", None, mll, depth, n_extra)
    x = _images(cfg, 6, 12)
    with torch.inference_mode():
        labels, scores, maps = m.beam_search(x, K, return_attention=True)
        labels0, scores0 = m.beam_search(x, K)
        ids_m = m.model.beam_search(x, K, return_attention=True)
        ids_0 = m.model.beam_search(x, K)
    assert labels == labels0 and torch.equal(scores, scores0)
    for a, b in zip(ids_m[:3], ids_0):
        assert torch.equal(a, b)
    S = maps.shape[2]
    # a hypothesis of S characters ended without EOS: no label to score, every row is its own
    cands = [[h if len(h) <= mll else "" for h in hyps] for hyps in labels]
    _, _, sm = _score(m, x, cands)
    checked = 0
    for b, hyps in enumerate(labels):
        for k in range(K):
            if k >= len(hyps):
                assert not bool(maps[b, k].any())
                continue
            n = len(hyps[k])
            if n > mll:
                continue
            assert torch.equal(maps[b, k, :n + 1], sm[b, k, :n + 1]), (b, k, hyps[k])
            assert not bool(maps[b, k, n + 1:].any())
            checked += 1
    assert checked >= K, labels
    if K == 1:
        with torch.inference_mode():
            logits, read = m.read_with_attention(x)
        greedy, _ = m.postprocess(logits)
        for b, lab in enumerate(greedy):
            if labels[b] and labels[b][0] == lab and len(lab) <= mll:
                assert torch.equal(maps[b, 0, :len(lab) + 1], read[b, :len(lab) + 1])
    assert S == mll + 1


def test_lexicon_maps_are_the_score_maps_of_the_chosen_word():
    cfg, _, m = _model()
    x = _images(cfg, 5, 13)
    lex = _words(cfg, 40, 3, 8) + ["", "a"]
    with torch.inference_mode():
        lab_b, lp_b, maps_b = m.lexicon_decode(x, lex, beam_width=4, return_attention=True)
        lab_s, lp_s, maps_s = m.lexicon_decode(x, lex, return_attention=True)
        lab_b0, lp_b0 = m.lexicon_decode(x, lex, beam_width=4)
    assert lab_b == lab_b0 and torch.equal(lp_b, lp_b0)
    words = [[w if w is not None else ""] for w in lab_b]
    _, _, sm = _score(m, x, words)
    for b, w in enumerate(lab_b):
        if w is None:
            assert not bool(maps_b[b].any())
            continue
        assert torch.equal(maps_b[b, :len(w) + 1], sm[b, 0, :len(w) + 1])
        if lab_s[b] == w:
            assert torch.equal(maps_s[b], sm[b, 0])


# ---- invariance and nothing else changes ---------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 10, 100])
def test_maps_do_not_depend_on_the_neighbours(K):
    cfg, _, m = _model()
    x = _images(cfg, 5, 14)
    mine = _words(cfg, 6, 21)
    alone = _score(m, x[:1], [mine])
    for i, others in enumerate([[["x"]] * 4, [_words(cfg, K, 30 + j) for j in range(4)]]):
        got = _score(m, x, [mine] + others)
        for a, b in zip(alone, got):
            assert torch.equal(a[0], b[0][:len(mine)]), i
    with torch.inference_mode():
        no_maps = m.score(x, [mine] + [_words(cfg, K, 40 + j) for j in range(4)], return_token_logprobs=True)
    with_maps = _score(m, x, [mine] + [_words(cfg, K, 40 + j) for j in range(4)])
    assert torch.equal(no_maps[0], with_maps[0]) and torch.equal(no_maps[1], with_maps[1])


def test_maps_do_not_depend_on_group_and_super_chunk_splits():
    from parseq_b200.factory import create_model
    cfg, sd, m = _model()
    x = _images(cfg, 9, 15)
    cands = [_words(cfg, 3 + 7 * b, 50 + b) for b in range(9)]
    want = _score(m, x, cands)
    with torch.inference_mode():
        beam_want = m.model.beam_search(x, 3, return_attention=True)
    m2 = create_model("parseq", charset_train=cfg.charset_train, max_label_length=cfg.max_label_length, enc_depth=2)
    m2.model.load_state_dict(sd)
    m2 = m2.eval().to("cuda")
    m2.model.set_engine_option("max_batch", 4)     # three super-chunks; dec_chunk follows it down to 4: one image
    m2.model.set_engine_option("dec_chunk", 4)     # of beam rows, or up to 4 * 26 candidate rows, per group
    got = _score(m2, x, cands)
    for a, b in zip(want, got):
        assert torch.equal(a, b)
    with torch.inference_mode():
        beam_got = m2.model.beam_search(x, 3, return_attention=True)
    for a, b in zip(beam_want, beam_got):
        assert torch.equal(a, b)
    m2.model._engine.close()


def test_maps_are_the_same_for_crops_and_their_uint8_stack():
    cfg, _, m = _model()
    g = torch.Generator().manual_seed(3)
    crops = [torch.randint(0, 256, (int(h), int(w), 3), generator=g, dtype=torch.uint8).cuda()
             for h, w in ((20, 70), (40, 90), (33, 33))]
    rot = [0, 90, 270]
    cands = [_words(cfg, 4, 60 + b) for b in range(3)]
    with torch.inference_mode():
        u8 = m.preprocess(crops, rotation=rot)
    a = _score(m, crops, cands, rotation=rot)
    b = _score(m, u8, cands)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    with torch.inference_mode():
        ba = m.model.beam_search(crops, 3, rotation=rot, return_attention=True)
        bb = m.model.beam_search(u8, 3, return_attention=True)
    for u, v in zip(ba, bb):
        assert torch.equal(u, v)


# ---- accuracy against the fp64 rounding-point maps -----------------------------------------------------------------
ACC_CASES = [("parseq", None, 25, 1, 0), ("parseq", None, 25, 2, 0), ("parseq", None, 63, 1, 0),
             ("parseq-tiny", None, 25, 1, 2906), ("parseq-tiny", None, 25, 1, 16289), ("parseq", 32, 25, 1, 0),
             ("parseq", 65, 25, 1, 0), ("parseq", 130, 25, 1, 0), ("parseq", 256, 25, 1, 0),
             ("parseq-patch16-224", None, 25, 1, 0)]


@pytest.mark.parametrize("case", ACC_CASES, ids=[f"{e}-T{t}-mll{m}-d{d}-x{n}" for e, t, m, d, n in ACC_CASES])
def test_score_maps_within_rounding_point_bound(case):
    exp, T, mll, depth, n_extra = case
    cfg, sd, m = _model(exp, T, mll, depth, n_extra)
    B = 3
    x = _images(cfg, B, 16)
    cands = [_words(cfg, 3, 70 + b) for b in range(B)]
    _, _, maps = _score(m, x, cands)
    with torch.inference_mode():
        mem = m.model.encode(x)
    from parseq_b200.system import pack_candidates
    targets, lengths, _ = pack_candidates(m.tokenizer, cands, B, mll, cfg.num_classes)
    ref = MapsReference(cfg, sd, device="cuda")
    got, want = [], []
    mi = 0
    for b in range(B):
        for k in range(len(cands[b])):
            n = int(lengths[mi])
            w = ref.ar(mem[b:b + 1], targets[mi:mi + 1])[0]
            got.append(_flat(maps[b, k])[:n + 1])
            want.append(w[:n + 1])
            assert not bool(maps[b, k, n + 1:].any())
            mi += 1
    got, want = torch.cat(got), torch.cat(want)
    assert bool((got >= 0).all()) and float((got.double().sum(-1) - 1).abs().max()) <= 1e-5
    s = map_stats(got, want)
    print(format_stats(f"[{exp} T{cfg.num_patches} mll{mll} d{depth} C{cfg.num_classes}]", s))
    assert max(excess(s, BOUNDS).values()) <= 1.0, (s, BOUNDS)


# ---- against the reference's own maps (tests/golden/alignment, tests/make_golden_alignment.py) -----------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "alignment")
GOLDENS = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.endswith(".pt")) if os.path.isdir(GOLDEN) else []


@pytest.mark.parametrize("name", GOLDENS)
def test_score_maps_against_goldens(name):
    """Every candidate's rows 0..n within GOLDEN_BOUNDS of the fp64 reference's (its ids are given: no margin filter)."""
    from make_golden_alignment import golden_case
    from parseq_b200.factory import create_model
    blob, cfg, sd, x, targets, lengths, per_image = golden_case(name)
    m = create_model(blob["experiment"], charset_train=cfg.charset_train, max_label_length=cfg.max_label_length,
                     img_size=cfg.img_size, dec_depth=cfg.dec_depth)
    m.model.load_state_dict(sd)
    m = m.eval().to("cuda")
    with torch.inference_mode():
        _, maps = m.model.score(x.cuda(), targets, lengths, per_image, return_attention=True)
    got = torch.cat([maps[i, :int(n) + 1] for i, n in enumerate(lengths.tolist())])
    s = map_stats(got, blob["maps"])
    print(format_stats(name, s))
    assert max(excess(s, GOLDEN_BOUNDS).values()) <= 1.0, (s, GOLDEN_BOUNDS)
    m.model._engine.close()


# ---- the cross-attention probe (tests/probe_models.py) ------------------------------------------------------------
@pytest.mark.parametrize("T", [32, 65, 130, 240, 256])
def test_grouped_maps_kernel_on_the_cross_attention_probe(T):
    """dec_cross's head 0 puts its weight on the last image token (score -64 against -256 for the others), so a phantom
    key T (a zero key, score 0) takes head 0's 1 / 12 of every row's mass and a dropped last key spreads it over the
    others.  The batch puts a
    seeded image between two probe images, with 1, 9 and 4 candidates: a CTA reading a neighbour's K gives one image
    the other's maps.  Each image's rows are held to 1e-4 of the fp64 rounding-point maps fed its own bf16 memory."""
    import probe_models as pm
    from parseq_b200.factory import create_model
    from parseq_b200.system import pack_candidates
    from parseq_b200.weights import synth_images
    p = pm.dec_cross((384, 1), T)
    m = create_model(pm.EXPERIMENT[384], **{**p.over, "dec_depth": 1})
    m.model.load_state_dict(p.sd)
    m = m.eval().to("cuda")
    m.model.set_engine_option("fuse_ln", 0)
    x = torch.cat([p.images[:1], synth_images(p.cfg, 1, 19), p.images[1:2]]).cuda()
    cands = [_words(p.cfg, 1, 90), _words(p.cfg, 9, 91), _words(p.cfg, 4, 92)]
    targets, lengths, per_image = pack_candidates(m.tokenizer, cands, 3, p.cfg.max_label_length, p.cfg.num_classes)
    with torch.inference_mode():
        mem = m.model.encode(x).to(torch.bfloat16).float()
        _, maps = m.model.score(x, targets, lengths, per_image, return_attention=True)
    ref = MapsReference(p.cfg, p.sd, device="cuda")
    img = torch.repeat_interleave(torch.arange(3), per_image.long())
    worst = 0.0
    for i, n in enumerate(lengths.tolist()):
        b = int(img[i])
        want = ref.ar(mem[b:b + 1], targets[i:i + 1])[0, :n + 1]
        worst = max(worst, float((maps[i, :n + 1].double() - want.to(maps.device)).abs().max()))
        assert not bool(maps[i, n + 1:].any())
    print(f"[dec_cross T{T}] max |engine - model| {worst:.2e}")
    assert worst <= 1e-4, worst
    m.model._engine.close()


# ---- resources and locate(text=) -----------------------------------------------------------------------------------
def test_calls_with_maps_release_everything():
    from parseq_b200.engine import load_library
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    lib = load_library()

    def counters():
        gc.collect()
        torch.cuda.synchronize()
        return int(lib.parseq_debug_int(None, b"live_device_bytes")), int(lib.parseq_debug_int(None, b"live_cuda_objects"))

    cfg, sd, _ = _model(depth=2)
    base = counters()
    m = create_model("parseq", charset_train=cfg.charset_train, enc_depth=2, dec_depth=2)
    m.model.load_state_dict(sd)
    m = m.eval().to("cuda")
    x = _images(cfg, 4, 17)
    with torch.inference_mode():
        m.score(x, _words(cfg, 12, 80), return_attention=True)
        m.beam_search(x, 5, return_attention=True)
        m.lexicon_decode(x, _words(cfg, 30, 81, 6), beam_width=3, return_attention=True)
        m.locate(x, text="abc")
    assert counters() != base
    m.model._engine.close()
    del m
    assert counters() == base


@pytest.mark.parametrize("crops", [False, True], ids=["tensor", "rotated_crops"])
def test_locate_text_of_the_greedy_reading_is_locate(crops):
    cfg, _, m = _model()
    if crops:
        g = torch.Generator().manual_seed(4)
        x = [torch.randint(0, 256, (int(h), int(w), 3), generator=g, dtype=torch.uint8).cuda()
             for h, w in ((24, 80), (90, 30), (40, 100), (64, 64))]
        rot = [0, 90, 180, 270]
    else:
        x, rot = _images(cfg, 5, 18), 0
    with torch.inference_mode():
        labels, _, c0, b0 = m.locate(x, rotation=rot)
    keep = [b for b, lab in enumerate(labels) if len(lab) <= cfg.max_label_length]
    assert len(keep) >= 3, labels
    x = [x[b] for b in keep] if crops else x[keep]
    rot = [rot[b] for b in keep] if crops else 0
    labels, c0, b0 = [labels[b] for b in keep], [c0[b] for b in keep], [b0[b] for b in keep]
    with torch.inference_mode():
        texts, lp, c1, b1 = m.locate(x, rotation=rot, text=labels)
        want = m.score(x, [[t] for t in labels], rotation=rot)[:, 0]
    assert texts == labels
    assert torch.equal(lp, want)
    for b in range(len(labels)):
        assert torch.equal(c0[b], c1[b]) and torch.equal(b0[b], b1[b]), b
