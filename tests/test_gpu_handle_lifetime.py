"""GPU: one engine handle across a lifetime of calls.

A long-lived handle (a server with mixed traffic, a validation loop that changes the weights between calls) keeps
state from call to call: CUDA graphs keyed by the call's shape and schedule, buffers allocated or grown on first use
(attention maps, scoring metadata, beam and lexicon buffers, lexicon roots, the host-crop staging buffer), options
that drop the graphs or reallocate the workspace, and the tables parseq_finalize derives from the weights.  Every
test here compares a call on a used handle with the same call on a fresh model that has the same weights and options
and runs that call alone.  The comparison is bitwise (torch.equal; floats as their bits, so -inf padding and NaN
fill compare too): DESIGN.md §5 makes graph replay equal eager, and a row's bits independent of the batch within a
kernel regime, and the same batch always picks the same regime.

Encoders have depth 2, as in the isolation tests: the fresh-model correctness of each call is tested elsewhere."""
import gc
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")

# kind -> (experiment, extra characters (head classes 95 + n), dec_depth)
KINDS = {
    "s95": ("parseq", 0, 1),
    "s195": ("parseq", 100, 1),          # > 128 classes: the class-sliced head and the top-K epilogue
    "d2": ("parseq", 0, 2),
    "tiny": ("parseq-tiny", 0, 1),
    "vitstr": ("vitstr", 0, 1),
}

_SD = {}


def _cfg_sd(kind, seed):
    from make_golden_long import charset
    from parseq_b200.config import make_config
    from parseq_b200.weights import init_state_dict
    exp, n_extra, depth = KINDS[kind]
    over = dict(charset_train=charset(n_extra), enc_depth=2)
    if exp != "vitstr":
        over["dec_depth"] = depth
    cfg = make_config(exp, **over)
    if (kind, seed) not in _SD:
        _SD[(kind, seed)] = init_state_dict(cfg, seed)
    return cfg, _SD[(kind, seed)]


def build(kind, seed=0, options=(), sd=None, inference=False):
    """A system of `kind` on the weights of `seed` (or `sd`), on cuda, with `options` ((name, value) pairs, applied in
    order) set; with `inference` built and loaded under torch.inference_mode (inference-tensor parameters)."""
    from parseq_b200.factory import create_model
    from parseq_b200.system import VitstrModel
    cfg, sd0 = _cfg_sd(kind, seed)
    exp = KINDS[kind][0]
    with torch.inference_mode(inference):
        if exp == "vitstr":                  # the ViTSTR system pins depth 12: swap in a depth-2 model
            m = create_model("vitstr", charset_train=cfg.charset_train)
            m.model = VitstrModel(cfg)
        else:
            m = create_model(exp, charset_train=cfg.charset_train, enc_depth=2, dec_depth=cfg.dec_depth)
        m.model.load_state_dict(sd if sd is not None else sd0)
        m = m.eval().to("cuda")
    for name, value in options:
        m.model.set_engine_option(name, value)
    return m


def release(*models):
    for m in models:
        if m.model._engine is not None:
            m.model._engine.close()
    gc.collect()


# ---------------------------------------------------------------- comparison

def _host(v):
    if isinstance(v, torch.Tensor):
        return v.detach().cpu()
    if isinstance(v, (list, tuple)):
        return type(v)(_host(u) for u in v)
    return v


def same(a, b):
    """Bitwise equality of nested outputs (floats as their bits)."""
    if isinstance(a, torch.Tensor):
        if not isinstance(b, torch.Tensor) or a.dtype != b.dtype or a.shape != b.shape:
            return False
        if a.is_floating_point():
            a, b = a.contiguous().view(torch.int32 if a.element_size() == 4 else torch.int16), b.contiguous().view(
                torch.int32 if b.element_size() == 4 else torch.int16)
        return torch.equal(a, b)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same(u, v) for u, v in zip(a, b))
    return a == b


def run(m, call):
    with torch.inference_mode():
        out = call(m)
    torch.cuda.synchronize()
    return _host(out)


# ---------------------------------------------------------------- inputs and calls

def _u8(cfg, B, seed):
    g = torch.Generator().manual_seed(seed)
    H, W = cfg.img_size
    return torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)


def _float(u8):
    return u8.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5).contiguous()


def _crops(B, seed, big=False):
    g = torch.Generator().manual_seed(seed)
    out = [torch.randint(0, 256, (20 + 7 * (i % 5), 60 + 13 * (i % 7), 3), generator=g, dtype=torch.uint8)
           for i in range(B)]
    if big:                                   # one 8192 x 3 crop: the host staging buffer grows
        out[0] = torch.randint(0, 256, (8192, 3, 3), generator=g, dtype=torch.uint8)
    return out


def _words(cs, k, seed, longest=10):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(k):
        n = int(torch.randint(1, longest + 1, (1,), generator=g))
        out.append("".join(cs[int(i)] for i in torch.randint(0, len(cs), (n,), generator=g)))
    return out


def forward(entry, B, seed, max_length=None, ar=True, refine=1, allow=None, maps=False, big=False):
    """A forward call through one of the six C entry points: (logits, ids, steps, maps), outputs filled with NaN / -7
    beforehand; with AR, no refinement and no max_length only the `steps` the call ran are compared."""
    def call(m):
        from parseq_b200.system import _crops_c, pack_crops
        cfg, eng = m.model.cfg, m.model.engine()
        host = entry.startswith("host")
        dev = torch.device("cpu") if host else torch.device("cuda")
        L = eng.num_steps(max_length)
        logits = torch.full((B, L, cfg.num_classes), NAN, device=dev, pin_memory=host)
        ids = torch.full((B, L), -7, dtype=torch.int32, device=dev, pin_memory=host)
        steps = torch.full((1,), -7, dtype=torch.int32, device=dev, pin_memory=host)
        amap = torch.full((B, L, cfg.enc_tokens), NAN, device=dev, pin_memory=host) if maps else None
        mask = m.allowlist_mask(allow, B) if allow is not None else None
        if mask is not None:
            mask = mask.pin_memory() if host else mask.cuda()
        kw = dict(class_mask_ptr=mask.data_ptr() if mask is not None else None,
                  attn_maps_ptr=amap.data_ptr() if maps else None)
        st = torch.cuda.current_stream().cuda_stream
        ptrs = (logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, max_length, ar, refine)
        u8 = _u8(cfg, B, seed)
        keep = []
        if entry == "float":
            keep.append(_float(u8).cuda())
            eng.forward(keep[0].data_ptr(), B, *ptrs, None, None, kw["class_mask_ptr"], kw["attn_maps_ptr"])
        elif entry == "host_float":
            keep.append(_float(u8).pin_memory())
            eng.forward_host(keep[0].data_ptr(), B, *ptrs, **kw)
        elif entry in ("u8", "host_u8"):
            keep.append(u8.pin_memory() if host else u8.cuda())
            eng.forward_u8(keep[0].data_ptr(), B, *ptrs, host=host, **kw)
        else:
            crops = _crops(B, seed, big)
            data, offsets, sizes = (pack_crops(crops, pin_memory=True) if host
                                    else pack_crops([c.cuda() for c in crops]))
            keep.append(data)
            eng.forward_crops(_crops_c(data, offsets, sizes, 0), B, *ptrs, host=host, **kw)
        torch.cuda.synchronize()
        out = [logits, ids, steps, amap]
        if ar and refine == 0 and max_length is None:
            S = int(steps[0])
            out = [logits[:, :S], ids[:, :S], steps, amap[:, :S] if maps else None]
        return out
    return call


def score(B, per, seed, shared=False, u8=False):
    def call(m):
        cs = m.model.cfg.charset_train
        cands = _words(cs, per, seed) if shared else [_words(cs, per, seed + b) for b in range(B)]
        imgs = _u8(m.model.cfg, B, seed)
        x = imgs.cuda() if u8 else _float(imgs).cuda()
        return m.score(x, cands, return_token_logprobs=True)
    return call


def beam(B, K, seed, max_length=None, allow=None, lexicon=None):
    """beam_search; `lexicon`: ("shared" | "per_image" | "compiled", words per list)."""
    def call(m):
        cs = m.model.cfg.charset_train
        x = _float(_u8(m.model.cfg, B, seed)).cuda()
        lex = None
        if lexicon is not None:
            how, k = lexicon
            if how == "per_image":
                lex = [_words(cs, k, seed + 100 + b) for b in range(B)]
            else:
                lex = _words(cs, k, seed + 100)
                if how == "compiled":
                    lex = m.compile_lexicon(lex)
        labels, scores = m.beam_search(x, K, max_length, allowlist=allow, lexicon=lex)
        return labels, scores
    return call


def encode(B, seed):
    return lambda m: m.model._features(_float(_u8(m.model.cfg, B, seed)).cuda())


def decode(B, J, seed):
    """encode, then decode with caller masks (padding, query and, at depth >= 2, content masks) and head."""
    def call(m):
        cfg = m.model.cfg
        g = torch.Generator().manual_seed(seed)
        mem = m.model.encode(_float(_u8(cfg, B, seed)).cuda())
        tgt = torch.randint(1, cfg.num_classes, (B, J), generator=g)
        tgt[:, 0] = cfg.num_tokens - 2                                       # BOS
        pad = torch.zeros((B, J), dtype=torch.bool)
        pad[0, J - 2:] = True
        causal = torch.triu(torch.ones((J, J), dtype=torch.bool), 1)
        qmask = causal.clone()
        qmask[1, 0] = True
        query = m.model.pos_queries[:, :J]
        y = m.model.decode(tgt.cuda(), mem, causal.cuda(), pad.cuda(), query, qmask.cuda())
        return y, m.model.head(y)
    return call


def text_embed(B, J, seed):
    def call(m):
        g = torch.Generator().manual_seed(seed)
        return m.model.text_embed(torch.randint(0, m.model.cfg.num_tokens, (B, J), generator=g).cuda())
    return call


def head(rows, seed):
    def call(m):
        g = torch.Generator().manual_seed(seed)
        return m.model.head(torch.randn((rows, m.model.cfg.embed_dim), generator=g).cuda())
    return call


def preprocess(B, seed):
    return lambda m: m.preprocess([c.cuda() for c in _crops(B, seed)])


def parseq_catalogue(cs):
    """(name, call) of the PARSeq catalogue; `cs`: the charset (allowlists are drawn from it)."""
    allow = cs[:20]
    per_image = [cs[5:30], None, cs[40:45], "", cs[:3], cs[60:90]]
    return [
        ("fwd_float_b300", forward("float", 300, 1)),                     # large, then small: stale static rows
        ("fwd_float_b3", forward("float", 3, 2)),
        ("fwd_u8_b5", forward("u8", 5, 3)),
        ("fwd_crops_b4", forward("crops", 4, 4)),
        ("fwd_host_float_b3", forward("host_float", 3, 5)),
        ("fwd_host_u8_b6", forward("host_u8", 6, 6)),
        ("fwd_host_crops_big_b3", forward("host_crops", 3, 7, big=True)),
        ("fwd_host_crops_b5", forward("host_crops", 5, 8)),
        ("fwd_ar0_b6", forward("float", 6, 9, refine=0)),                 # early exit: `steps`
        ("fwd_ar0_ml5_b6", forward("float", 6, 9, max_length=5, refine=0)),
        ("fwd_ar2_b6", forward("float", 6, 9, refine=2)),
        ("fwd_nar_b6", forward("float", 6, 9, ar=False)),
        ("fwd_ml7_b4", forward("float", 4, 10, max_length=7)),
        ("fwd_b700", forward("float", 700, 11)),                          # > max_batch: two super-chunks
        ("fwd_allow_b6", forward("float", 6, 12, allow=allow)),           # masked / unmasked at one batch
        ("fwd_noallow_b6", forward("float", 6, 12)),
        ("fwd_allow_per_image_b6", forward("float", 6, 12, allow=per_image)),
        ("fwd_host_u8_allow_b6", forward("host_u8", 6, 12, allow=allow)),
        ("maps_b5", forward("float", 5, 13, maps=True)),                  # maps on / off at one batch
        ("nomaps_b5", forward("float", 5, 13)),
        ("maps_ar0_b4", forward("float", 4, 14, refine=0, maps=True)),
        ("maps_nar_b4", forward("float", 4, 14, ar=False, maps=True)),
        ("maps_host_crops_b3", forward("host_crops", 3, 15, maps=True)),
        ("maps_b300", forward("float", 300, 16, maps=True, allow=allow)),
        ("score_many", score(6, 40, 17)),                                  # sc_meta growth, then a small call
        ("score_few", score(2, 2, 18)),
        ("score_shared_u8", score(5, 12, 19, shared=True, u8=True)),
        ("beam_k8", beam(4, 8, 20)),
        ("beam_k2", beam(4, 2, 20)),
        ("beam_k4_allow_ml6", beam(3, 4, 21, max_length=6, allow=allow)),
        ("lex_large", beam(4, 4, 22, lexicon=("shared", 300))),           # lex_roots / lexicon buffers
        ("lex_small", beam(4, 2, 22, lexicon=("shared", 5))),
        ("lex_per_image_large", beam(7, 3, 23, lexicon=("per_image", 60))),
        ("lex_per_image_small", beam(2, 3, 24, lexicon=("per_image", 4))),
        ("lex_compiled", beam(3, 5, 25, lexicon=("compiled", 40))),
        ("encode_b4", encode(4, 26)),
        ("decode_head_b3", decode(3, 9, 27)),
        ("head_rows", head(37, 28)),
        ("text_embed", text_embed(3, 11, 29)),
        ("preprocess_b4", preprocess(4, 30)),
    ]


def vitstr_catalogue(cs):
    allow = cs[:20]
    return [
        ("fwd_float_b300", forward("float", 300, 1, ar=False)),
        ("fwd_float_b3", forward("float", 3, 2, ar=False)),
        ("fwd_u8_b5", forward("u8", 5, 3, ar=False)),
        ("fwd_host_crops_big_b3", forward("host_crops", 3, 7, ar=False, big=True)),
        ("fwd_host_float_b4", forward("host_float", 4, 8, ar=False, max_length=9)),
        ("fwd_allow_b6", forward("float", 6, 12, ar=False, allow=allow)),
        ("fwd_noallow_b6", forward("float", 6, 12, ar=False)),
        ("fwd_b700", forward("float", 700, 11, ar=False)),
        ("score_many", score(6, 40, 17)),
        ("score_few", score(2, 2, 18)),
        ("beam_k8", beam(4, 8, 20)),
        ("beam_k2", beam(4, 2, 20)),
        ("lex_large", beam(4, 4, 22, lexicon=("shared", 300))),
        ("lex_small", beam(4, 2, 22, lexicon=("shared", 5))),
        ("lex_per_image_large", beam(7, 3, 23, lexicon=("per_image", 60))),
        ("lex_per_image_small", beam(2, 3, 24, lexicon=("per_image", 4))),
        ("encode_b4", encode(4, 26)),
    ]


def catalogue(kind):
    cfg, _ = _cfg_sd(kind, 0)
    return (vitstr_catalogue if kind == "vitstr" else parseq_catalogue)(cfg.charset_train)


def fresh(kind, call, seed=0, options=(), sd=None):
    """`call` alone on a fresh model."""
    m = build(kind, seed, options, sd)
    try:
        return run(m, call)
    finally:
        release(m)


def check(m, name, call, want):
    got = run(m, call)
    assert same(got, want), f"{name}: differs from the same call on a fresh model"


# ---------------------------------------------------------------- a. a catalogue of calls in several orders

@pytest.mark.parametrize("kind", ["s95", "s195", "d2", "vitstr"])
def test_catalogue_in_several_orders(kind):
    cat = catalogue(kind)
    refs = {name: fresh(kind, call) for name, call in cat}
    m = build(kind)
    bad = []
    orders = {"listed": list(cat), "reversed": list(reversed(cat))}
    for seed in (1, 2):
        shuffled = list(cat)
        random.Random(seed).shuffle(shuffled)
        orders[f"shuffle{seed}"] = shuffled
    for order, calls in orders.items():
        for name, call in calls:
            if not same(run(m, call), refs[name]):
                bad.append(f"{order}/{name}")
    release(m)
    assert not bad, f"calls on a used handle that differ from a fresh model: {bad}"


# ---------------------------------------------------------------- b. option changes between calls

OPTION_STEPS = [
    [("max_batch", 64)], [("max_batch", 512)], [("chunk", 3)], [("dec_chunk", 16)], [("dec_chunk", 128)],
    [("ar_kernel", 0)], [("ar_kernel", 1)], [("ar_kernel", 2)], [("ar_cluster_size", 6)], [("ar_cluster_size", 8)],
    [("ar_cluster_size", 0)], [("fuse_ln", 0)], [("fuse_ln", 3)], [("use_graph", 0)], [("use_graph", 1)],
]


def _probe(kind):
    """forward (large and small), score, beam and lexicon beam: what each option step is checked with."""
    cat = dict(catalogue(kind))
    return [(n, cat[n]) for n in ("fwd_float_b300", "fwd_float_b3", "score_many", "beam_k8", "lex_per_image_large")]


@pytest.mark.parametrize("kind", ["s95", "s195", "d2", "vitstr"])
def test_option_changes_between_calls(kind):
    from parseq_b200.engine import EngineError
    m = build(kind)
    for name, call in catalogue(kind):
        run(m, call)
    history = []
    bad = []
    for step in OPTION_STEPS:
        (opt, value), = step
        if kind == "vitstr" and opt.startswith("ar_"):
            continue
        try:
            m.model.set_engine_option(opt, value)
        except EngineError:
            # the grid-barrier AR kernel is refused where it cannot run (e.g. dec_depth 2): the handle keeps its options
            assert (opt, value) == ("ar_kernel", 1), (opt, value)
            continue
        history.append((opt, value))
        # the reference: one fresh model with the same options, running the probe calls in order
        ref = build(kind, options=history)
        for name, call in _probe(kind):
            if not same(run(m, call), run(ref, call)):
                bad.append(f"{opt}={value}/{name}")
        release(ref)
    release(m)
    assert not bad, f"calls after an option change that differ from a fresh model with those options: {bad}"


def test_process_default_options_reach_only_later_handles():
    """parseq_set_option(NULL, ...) sets the defaults of handles created afterwards: attn_impl = 1 (the wgmma attention
    core instead of the fused QKV + attention kernel) changes a call's launches and must leave an existing handle as
    it was."""
    from parseq_b200.engine import check as check_rc, load_library
    lib = load_library()
    call = forward("float", 4, 40)
    before = build("s95")
    eng = before.model.engine()
    want = run(before, call)
    n0 = eng.launches
    run(before, call)
    per_call = eng.launches - n0
    try:
        check_rc(lib, lib.parseq_set_option(None, b"attn_impl", 1))
        n0 = eng.launches
        assert same(run(before, call), want)
        assert eng.launches - n0 == per_call, "the process default reached a handle created before it was set"
        after = build("s95")
        ea = after.model.engine()
        got = run(after, call)
        n0 = ea.launches
        run(after, call)
        assert ea.launches - n0 != per_call, "a handle created after the default was set does not use it"
    finally:
        check_rc(lib, lib.parseq_set_option(None, b"attn_impl", 0))
    explicit = build("s95", options=[("attn_impl", 1)])
    assert same(got, run(explicit, call))
    release(before, after, explicit)


# ---------------------------------------------------------------- c. weight updates under captured graphs

def _warm_calls(kind):
    cat = dict(catalogue(kind))
    names = ["fwd_float_b300", "fwd_float_b3", "score_many", "beam_k8", "lex_large"]
    if kind != "vitstr":
        names.insert(2, "maps_b5")
    return [(n, cat[n]) for n in names]


def _both_modes(m, calls):
    out = {}
    for graph in (1, 0):
        m.model.set_engine_option("use_graph", graph)
        for name, call in calls:
            out[(graph, name)] = run(m, call)
    m.model.set_engine_option("use_graph", 1)
    return out


def _reference(kind, calls, seed=0, sd=None):
    m = build(kind, seed, sd=sd)
    try:
        return _both_modes(m, calls)
    finally:
        release(m)


def _switch(m, path, sd, delta_sign=0, delta=None):
    if path == "load_state_dict":
        m.model.load_state_dict(sd)
    elif path == "assign":
        m.model.load_state_dict({k: v.to("cuda") for k, v in sd.items()}, assign=True)
    elif path == "inference":
        with torch.inference_mode():
            m.model.load_state_dict(sd)
    else:
        with torch.no_grad():
            for k, p in m.model.named_parameters():
                if delta_sign:
                    p.add_(delta[k].to(p.device), alpha=delta_sign)
                else:
                    p.copy_(sd[k].to(p.device))


@pytest.mark.parametrize("path", ["load_state_dict", "assign", "inference", "inplace"])
@pytest.mark.parametrize("kind", ["s95", "d2", "vitstr"])
def test_weight_update_under_captured_graphs(kind, path):
    calls = _warm_calls(kind)
    _, sd0 = _cfg_sd(kind, 0)
    _, sd1 = _cfg_sd(kind, 1)
    m = build(kind, 0, inference=(path == "inference"))
    first = _both_modes(m, calls)
    if path == "inplace":                     # p.add_(sd1 - sd0) under no_grad: the reference gets the sums
        delta = {k: sd1[k] - sd0[k] for k in sd0}
        _switch(m, path, None, +1, delta)
        sd_new = {k: v.detach().cpu().clone() for k, v in m.model.state_dict().items()}
    else:
        _switch(m, path, sd1)
        sd_new = sd1
    second = _both_modes(m, calls)
    want = _reference(kind, calls, sd=sd_new)
    bad = [f"seed1/{'graph' if g else 'eager'}/{n}" for (g, n) in want if not same(second[(g, n)], want[(g, n)])]
    _switch(m, path, sd0)                     # back: the tables are rebuilt, not accumulated
    third = _both_modes(m, calls)
    bad += [f"seed0/{'graph' if g else 'eager'}/{n}" for (g, n) in first if not same(third[(g, n)], first[(g, n)])]
    assert not any(same(second[k], first[k]) for k in first if k[1].startswith("fwd")), "seed 1 changed nothing"
    ref0 = _reference(kind, calls[:2], seed=0)
    bad += [f"first/{k}" for k in ref0 if not same(first[k], ref0[k])]
    release(m)
    assert not bad, f"calls after a weight update that differ from a fresh model on those weights: {bad}"


# ---------------------------------------------------------------- d. rejected calls leave the handle as it was

def _rejected(kind):
    """(name, call that the host refuses, exception type) for `kind`."""
    from parseq_b200.engine import EngineError
    from parseq_b200.system import CropsC

    def wrong_mask(m):
        x = _float(_u8(m.model.cfg, 3, 50)).cuda()
        words = (m.model.cfg.num_classes + 31) // 32
        return m.model._run(x, None, True, 1, class_mask=torch.zeros((4, words), dtype=torch.int32))

    def long_word(m):
        x = _float(_u8(m.model.cfg, 3, 50)).cuda()
        return m.beam_search(x, 2, lexicon=["ab", m.model.cfg.charset_train[0] * (m.model.cfg.max_label_length + 1)])

    def beam_width(k):
        return lambda m: m.beam_search(_float(_u8(m.model.cfg, 2, 51)).cuda(), k)

    def bad_crops(m):
        eng = m.model.engine()
        data = torch.zeros(3 * 10 * 10, dtype=torch.uint8, device="cuda")
        offsets = torch.tensor([0, 300], dtype=torch.int64)           # crop 1 starts past the data
        sizes = torch.tensor([[10, 10], [10, 10]], dtype=torch.int32)
        out = torch.empty((2, 26, m.model.cfg.num_classes), device="cuda")
        ids = torch.empty((2, 26), dtype=torch.int32, device="cuda")
        steps = torch.empty((1,), dtype=torch.int32, device="cuda")
        eng.forward_crops(CropsC(data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), 0), 2,
                          out.data_ptr(), ids.data_ptr(), steps.data_ptr(), torch.cuda.current_stream().cuda_stream)

    def bad_rotation(m):
        from parseq_b200.system import _crops_c, pack_crops
        data, offsets, sizes = pack_crops([c.cuda() for c in _crops(2, 52)])
        eng = m.model.engine()
        out = torch.empty((2, 26, m.model.cfg.num_classes), device="cuda")
        ids = torch.empty((2, 26), dtype=torch.int32, device="cuda")
        steps = torch.empty((1,), dtype=torch.int32, device="cuda")
        eng.forward_crops(_crops_c(data, offsets, sizes, 45), 2, out.data_ptr(), ids.data_ptr(), steps.data_ptr(),
                          torch.cuda.current_stream().cuda_stream)

    def engine_forward(m, forced=False, mask=False, maps=False):
        """parseq_forward itself with the combination the host must refuse."""
        cfg, eng = m.model.cfg, m.model.engine()
        x = _float(_u8(cfg, 2, 53)).cuda()
        L = eng.num_steps(None)
        out = torch.empty((2, L, cfg.num_classes), device="cuda")
        ids = torch.empty((2, L), dtype=torch.int32, device="cuda")
        steps = torch.empty((1,), dtype=torch.int32, device="cuda")
        f = torch.zeros((2, L), dtype=torch.int32, device="cuda")
        w = torch.full((2, (cfg.num_classes + 31) // 32), -1, dtype=torch.int32, device="cuda")
        a = torch.empty((2, L, cfg.enc_tokens), device="cuda")
        eng.forward(x.data_ptr(), 2, out.data_ptr(), ids.data_ptr(), steps.data_ptr(),
                    torch.cuda.current_stream().cuda_stream, None, True, 1, f.data_ptr() if forced else None, None,
                    w.data_ptr() if mask else None, a.data_ptr() if maps else None)

    def mask_and_forcing(m):
        x = _float(_u8(m.model.cfg, 2, 53)).cuda()
        words = (m.model.cfg.num_classes + 31) // 32
        return m.model._run(x, None, True, 1, forced_ids=torch.zeros((2, 26), dtype=torch.int32),
                            class_mask=torch.zeros((2, words), dtype=torch.int32))

    out = [("wrong_allowlist_shape", wrong_mask, ValueError), ("over_long_lexicon_word", long_word, ValueError),
           ("beam_width_0", beam_width(0), ValueError), ("beam_width_17", beam_width(17), ValueError),
           ("crop_past_data", bad_crops, EngineError), ("crop_rotation_45", bad_rotation, EngineError)]
    if kind == "vitstr":
        out += [("vitstr_maps", lambda m: m.read_with_attention(_float(_u8(m.model.cfg, 2, 54)).cuda()),
                 NotImplementedError),
                ("vitstr_maps_engine", lambda m: engine_forward(m, maps=True), EngineError)]
    else:
        out += [("mask_with_forcing", mask_and_forcing, ValueError),
                ("mask_with_forcing_engine", lambda m: engine_forward(m, forced=True, mask=True), EngineError),
                ("maps_with_forcing_engine", lambda m: engine_forward(m, forced=True, maps=True), EngineError)]
    return out


@pytest.mark.parametrize("kind", ["s95", "vitstr"])
def test_rejected_calls_leave_the_handle_as_it_was(kind):
    good = [(n, c) for n, c in catalogue(kind) if n in ("fwd_float_b3", "fwd_float_b300", "score_few", "beam_k2",
                                                       "lex_small", "fwd_host_crops_big_b3", "maps_b5")]
    refs = {n: fresh(kind, c) for n, c in good}
    m = build(kind)
    eng = m.model.engine()
    bad = []
    for i, (name, call, exc) in enumerate(_rejected(kind)):
        gname, gcall = good[i % len(good)]
        check(m, gname, gcall, refs[gname])
        torch.cuda.synchronize()
        n0 = eng.launches
        with pytest.raises(exc):
            with torch.inference_mode():
                call(m)
        torch.cuda.synchronize()
        if eng.launches != n0:
            bad.append(f"{name} launched {eng.launches - n0} kernels")
        gname, gcall = good[(i + 1) % len(good)]
        if not same(run(m, gcall), refs[gname]):
            bad.append(f"{gname} after {name}")
    release(m)
    assert not bad, bad


# ---------------------------------------------------------------- e. two handles in one process

def test_two_handles_interleaved_on_several_streams():
    """PARSeq-S with small decoder chains and parseq-tiny in eager mode, plus ViTSTR, each call interleaved with the
    others' on the current stream and on two user streams: each result equals that model's solo reference."""
    setups = {"s95": [("dec_chunk", 32)], "tiny": [("use_graph", 0), ("fuse_ln", 0)], "vitstr": [("chunk", 64)]}
    picks = ("fwd_float_b300", "fwd_float_b3", "fwd_host_u8_b6", "score_many", "beam_k8", "lex_large", "maps_b5")
    work = []
    for kind in setups:
        work += [(kind, n, c) for n, c in catalogue(kind) if n in picks]
    refs = {(k, n): fresh(k, c, options=setups[k]) for k, n, c in work}
    models = {k: build(k, options=o) for k, o in setups.items()}
    streams = [None, torch.cuda.Stream(), torch.cuda.Stream()]
    order = work * 2
    random.Random(3).shuffle(order)
    bad = []
    for i, (kind, name, call) in enumerate(order):
        s = streams[i % 3]
        torch.cuda.synchronize()
        with torch.cuda.stream(s) if s is not None else torch.cuda.stream(torch.cuda.current_stream()):
            with torch.inference_mode():
                out = call(models[kind])
        torch.cuda.synchronize()
        if not same(_host(out), refs[(kind, name)]):
            bad.append(f"{i}:{kind}/{name}/stream{i % 3}")
    release(*models.values())
    assert not bad, f"interleaved calls that differ from the model's solo reference: {bad}"
