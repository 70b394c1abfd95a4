"""GPU: the decoder on its own, against the fp64 rounding-point model of tests/decoder_reference.py.

Every case builds a model with sharp (x4) attention weights and the unfused encoder LayerNorm (fuse_ln = 0), takes the
engine's own encoder memory from `encode` (the fp32 output of the LayerNorm whose bf16 copy the decoder reads), runs
`forward` under teacher forcing (`forced_ids` / `forced_refine`, so every AR step and refinement pass is a fixed function
of the memory and its context), and compares the logits with the model fed bf16(memory), computed in fp64 on the GPU.
Without the encoder's bf16 cascade in the comparison, the engine is held to decoder_reference.BOUNDS, which
tests/test_decoder_budget_cpu.py places at least 2x above the fp32 stand-in's noise and at least 2x below each injected
decoder bug, save the small bugs it names at D >= 384 and at depth 2.  The cases reach every AR instantiation the dispatcher can pick, by name, the grid-barrier kernel and the
chain, the head widths at their edges, the image-token counts at the edges of the K/V boxes, and the NAR, refinement,
`decode` and depth-2 passes.  Each case prints its statistics (run with -s to see them)."""
import pytest
import torch

from decoder_reference import (BOUNDS, DecoderReference, DepthDecoderReference, budget_stats, excess, forced_ar_ids,
                               format_stats, refine_context)
from make_golden_long import charset
from token_count_geometries import geometry_config

pytestmark = pytest.mark.gpu

WIDTHS = {192: "parseq-tiny", 384: "parseq", 768: "parseq-base-48x160"}
WIDE_EXTRA = 100                      # 195 head classes: the class-sliced head (> 128)
_MODELS = {}


def _model(D, mll=25, chars=None, T=None, depth=1):
    """(config, state_dict, model) with a depth-2 encoder; cached, a few at a time."""
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    key = (D, mll, chars, T, depth)
    if key not in _MODELS:
        if len(_MODELS) >= 3:
            _MODELS.clear()
        exp = WIDTHS[D]
        over = dict(geometry_config(T, exp)[1]) if T is not None else dict(enc_depth=2)
        over.update(charset_train=chars if chars is not None else charset(0), max_label_length=mll, dec_depth=depth)
        cfg = make_config(exp, **over)
        sd = init_state_dict(cfg, 21, sharp=4.0)
        m = create_model(exp, **over)
        m.model.load_state_dict(sd)
        m = m.eval().to("cuda")
        m.model.set_engine_option("max_batch", 64)
        _MODELS[key] = (cfg, sd, m)
    cfg, sd, m = _MODELS[key]
    for k, v in (("fuse_ln", 0), ("ar_kernel", 2), ("ar_cluster_size", 0), ("ar_clusters", 0)):
        m.model.set_engine_option(k, v)
    return cfg, sd, m


def _check(name, D, got, ref, depth=1):
    s = budget_stats(got, ref)
    print(format_stats(f"[{name}] D {D}", s))
    assert max(excess(s, (D, depth)).values()) <= 1.0, (name, s, BOUNDS[(D, depth)])


def _forward(cfg, sd, m, B, *, seed=0, ar=True, refine=0, first_eos=(1, 5, 12, 20, 25, None), opts=(), depth=1):
    """Runs the engine under teacher forcing and returns (engine logits, fp64 model logits of the same pass)."""
    from parseq_b200.weights import synth_images
    mll = cfg.max_label_length
    L, C, bos = mll + 1, cfg.num_classes, cfg.num_tokens - 2
    for k, v in opts:
        m.model.set_engine_option(k, v)
    m.model.decode_ar, m.model.refine_iters = ar, refine
    x = synth_images(cfg, B, 60 + seed).cuda()
    forced = forced_ar_ids(B, L, C, bos, 10 + seed) if ar else None
    fr = (torch.stack([refine_context(B, L, C, bos, first_eos, 20 + seed + r) for r in range(refine)])
          if refine else None)
    with torch.inference_mode():
        mem = m.model.encode(x)
        got = m.model.forward(m.tokenizer, x, mll, forced_ids=forced, forced_refine=fr)
    # the logits of an AR run come from the AR loop; the cluster kernel's cross-attention operands are hi + lo pairs
    cluster = ar and not refine and m.model.engine().debug_int("ar_last_path") == 2
    model = (DepthDecoderReference if depth > 1 else DecoderReference)(cfg, sd, device="cuda", cluster=cluster)
    if refine:
        ref = model.refine(mem, fr[-1])
    elif ar:
        ref = model.ar(mem, forced)
    else:
        ref = model.nar(mem, L)
    assert got.shape == ref.shape == (B, L, C)
    return got, ref


# ---- every cluster-kernel instantiation, by name ----------------------------------------------------------------------
# (MT, CS, head split) -> (batch, engine options); clusters of 4 (2) hold a batch of 40 (60) in one wave with one (two)
# m16 row tiles per cluster; at B <= 2 every image gets a cluster to itself, so (image, head pair) units fit one cluster
ROUTES = {
    (1, 8, 0): (40, (("ar_cluster_size", 8), ("ar_clusters", 4))),
    (1, 8, 1): (None, (("ar_cluster_size", 8),)),
    (2, 8, 0): (60, (("ar_cluster_size", 8), ("ar_clusters", 2))),
    (1, 6, 0): (40, (("ar_cluster_size", 6), ("ar_clusters", 4))),
    (2, 6, 0): (60, (("ar_cluster_size", 6), ("ar_clusters", 2))),
}
AR_CASES = [(D, r, wide, pitch) for D in (192, 384) for r in ROUTES for wide in (0, 1) for pitch in (32, 64)] + \
           [(768, r, wide, pitch) for r in ((1, 8, 0), (1, 6, 0)) for wide in (0, 1) for pitch in (32, 64)]


def _ar_id(c):
    D, (mt, cs, hs), wide, pitch = c
    return f"D{D}-mt{mt}-cs{cs}-hs{hs}-{'wide' if wide else 'c95'}-idp{pitch}"


@pytest.mark.parametrize("case", AR_CASES, ids=[_ar_id(c) for c in AR_CASES])
def test_cluster_ar_instantiation(case):
    D, (mt, cs, hs), wide, pitch = case
    cfg, sd, m = _model(D, 25 if pitch == 32 else 63, charset(WIDE_EXTRA if wide else 0))
    B, opts = ROUTES[(mt, cs, hs)]
    if B is None:
        B = 2 if D == 192 else 1
    got, ref = _forward(cfg, sd, m, B, opts=opts)
    eng = m.model.engine()
    reached = tuple(eng.debug_int(k) for k in ("ar_last_path", "ar_last_mt", "ar_last_cluster_size", "ar_last_head_split",
                                                "ar_last_wide", "ar_last_ids_pitch"))
    assert reached == (2, mt, cs, hs, wide, pitch), reached
    _check(_ar_id(case), D, got, ref)


# ---- the grid-barrier kernel and the chain ----------------------------------------------------------------------------
@pytest.mark.parametrize("D", [192, 384])
@pytest.mark.parametrize("n_extra", [0, 15], ids=["c95", "c110"])
def test_grid_barrier_ar_kernel(D, n_extra):
    """C = 95 with ar_kernel = 1; C = 110 (97..128 classes, L <= 32) is where the default dispatch picks it."""
    cfg, sd, m = _model(D, 25, charset(n_extra))
    got, ref = _forward(cfg, sd, m, 6, opts=(("ar_kernel", 1),) if n_extra == 0 else ())
    assert m.model.engine().debug_int("ar_last_path") == 1
    _check(f"grid-barrier C{cfg.num_classes}", D, got, ref)


@pytest.mark.parametrize("D", sorted(WIDTHS))
@pytest.mark.parametrize("mll", [25, 63])
def test_chain_ar_loop(D, mll):
    cfg, sd, m = _model(D, mll)
    got, ref = _forward(cfg, sd, m, 6, opts=(("ar_kernel", 0),))
    assert m.model.engine().debug_int("ar_last_path") == 0
    _check(f"chain L{mll + 1}", D, got, ref)


def test_chain_for_97_to_128_classes_with_long_labels():
    cfg, sd, m = _model(384, 63, charset(15))
    got, ref = _forward(cfg, sd, m, 6)
    assert m.model.engine().debug_int("ar_last_path") == 0          # the grid-barrier kernel serves L <= 32 only
    _check("chain C110 L64", 384, got, ref)


# ---- head widths at the edges -----------------------------------------------------------------------------------------
HEADS = {
    "c2": (384, "a", 40, ()),                                         # the smallest head the engine accepts
    "c96": (384, charset(1), 6, ()),                                  # the widest redundant head
    "c129_cs8": (384, charset(34), 20, (("ar_cluster_size", 8), ("ar_clusters", 2))),   # Cs = 24: CTAs 6, 7 own no class
    "c129_hs": (384, charset(34), 1, (("ar_cluster_size", 8),)),
    "c3001": (384, charset(2906), 6, ()),
    "c16384_d192": (192, charset(16383 - 94), 4, ()),
}


@pytest.mark.parametrize("name", list(HEADS))
def test_head_width(name):
    D, chars, B, opts = HEADS[name]
    cfg, sd, m = _model(D, 25, chars)
    got, ref = _forward(cfg, sd, m, B, opts=opts)
    eng = m.model.engine()
    assert eng.debug_int("ar_last_path") == 2
    assert eng.debug_int("ar_last_wide") == (1 if cfg.num_classes > 128 else 0)
    if "cs8" in name:
        assert eng.debug_int("ar_last_cluster_size") == 8 and eng.debug_int("ar_last_head_split") == 0
    _check(f"head {name} C{cfg.num_classes}", D, got, ref)


# ---- image-token counts -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["cluster", "chain"])
@pytest.mark.parametrize("T", [32, 64, 65, 128, 130, 256])
def test_image_token_count(T, route):
    cfg, sd, m = _model(384, 25, T=None if T == 128 else T)
    assert cfg.num_patches == T
    got, ref = _forward(cfg, sd, m, 20, opts=(("ar_kernel", 0 if route == "chain" else 2),))
    assert m.model.engine().debug_int("ar_last_path") == (0 if route == "chain" else 2)
    _check(f"T{T} {route}", 384, got, ref)


# ---- the other decoder passes -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", sorted(WIDTHS))
def test_nar_pass(D):
    cfg, sd, m = _model(D, 25)
    got, ref = _forward(cfg, sd, m, 6, ar=False)
    _check("nar", D, got, ref)


@pytest.mark.parametrize("D", sorted(WIDTHS))
@pytest.mark.parametrize("mll", [25, 63])
def test_refine_pass_with_the_first_eos_in_either_key_group(D, mll):
    """First EOS at 1, 31, 32, 33 and 63, or absent: both 32-key ballot groups of the cloze mask's padding."""
    cfg, sd, m = _model(D, mll)
    got, ref = _forward(cfg, sd, m, 6, refine=1, first_eos=(1, 31, 32, 33, 63, None) if mll == 63 else (1, 2, 13, 25, None))
    _check(f"refine L{mll + 1}", D, got, ref)


def test_two_refine_passes():
    cfg, sd, m = _model(384, 25)
    got, ref = _forward(cfg, sd, m, 6, refine=2, seed=3)
    _check("refine_iters 2", 384, got, ref)


@pytest.mark.parametrize("depth", [1, 2])
def test_decode_api_with_masks(depth):
    """`model.decode` (parseq_decode_ex) on the engine memory: own queries, a query mask, a padding mask and, at depth 2,
    a content mask; the logits through `model.head`."""
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(384, 25, depth=depth)
    B, J, NQ, D = 4, 20, 26, 384
    g = torch.Generator().manual_seed(30 + depth)
    x = synth_images(cfg, B, 70).cuda()
    tgt = torch.randint(0, cfg.num_classes, (B, J), generator=g)
    tgt[:, 0] = cfg.num_tokens - 2
    tgt[:, 7] = cfg.num_classes - 1
    query = torch.randn((1, NQ, D), generator=g) * 0.1
    qmask = torch.rand((NQ, J), generator=g) < 0.3
    qmask[:, 0] = False
    pmask = torch.rand((B, J), generator=g) < 0.2
    pmask[:, 0] = False
    cmask = torch.triu(torch.ones((J, J), dtype=torch.bool), 1)
    cmask[5, 2] = True
    with torch.inference_mode():
        mem = m.model.encode(x)
        out = m.model.decode(tgt.cuda(), mem, tgt_mask=cmask.cuda(), tgt_padding_mask=pmask.cuda(),
                             tgt_query=query.cuda(), tgt_query_mask=qmask.cuda())
        got = m.model.head(out)
    model = (DepthDecoderReference if depth > 1 else DecoderReference)(cfg, sd, device="cuda")
    q = query.to("cuda", torch.float64).expand(B, -1, -1)
    dev = lambda t: t.cuda()
    if depth > 1:
        ref = model._decode(dev(tgt), model._memory(mem), q, dev(qmask), dev(pmask), dev(cmask))
    else:
        ref = model._decode(dev(tgt), model._memory(mem), q, dev(qmask), dev(pmask))
    assert got.shape == ref.shape == (B, NQ, cfg.num_classes)
    _check(f"decode depth {depth}", D, got, ref, depth)


@pytest.mark.parametrize("ar,refine", [(True, 0), (True, 1), (False, 0)], ids=["ar", "refine", "nar"])
def test_depth2_decoder_on_the_chain(ar, refine):
    cfg, sd, m = _model(384, 25, depth=2)
    got, ref = _forward(cfg, sd, m, 6, ar=ar, refine=refine, depth=2)
    if ar:
        assert m.model.engine().debug_int("ar_last_path") == 0
    _check(f"depth 2 {'refine' if refine else 'ar' if ar else 'nar'}", 384, got, ref, 2)


# ---- what the comparison rests on -------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", sorted(WIDTHS))
def test_encode_is_batch_invariant_and_forced_runs_replay(D):
    """`encode` gives an image the same memory alone and inside a batch (so the memory the model is fed is the one the
    forward pass decoded from), and a teacher-forced forward equals itself on replay."""
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(D, 25)
    x = synth_images(cfg, 6, 80).cuda()
    forced = forced_ar_ids(6, 26, cfg.num_classes, cfg.num_tokens - 2, 81)
    m.model.decode_ar, m.model.refine_iters = True, 0
    with torch.inference_mode():
        full = m.model.encode(x)
        for lo, hi in ((0, 1), (2, 5), (5, 6)):
            assert torch.equal(m.model.encode(x[lo:hi]), full[lo:hi])
        a = m.model.forward(m.tokenizer, x, 25, forced_ids=forced)
        b = m.model.forward(m.tokenizer, x, 25, forced_ids=forced)
    assert torch.equal(a, b)
