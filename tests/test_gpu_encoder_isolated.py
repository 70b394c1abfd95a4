"""GPU: the encoder on its own, against the fp64 rounding-point model of tests/encoder_reference.py.

Every case builds a model with sharp (x4) attention weights at encoder depth 1 or 2, runs `encode` (PARSeq) or
`forward_features` / `forward_tokens` (ViTSTR) under the launch options of one route, and compares the output with the
model computed in fp64 on the GPU, against encoder_reference.BOUNDS, which tests/test_encoder_budget_cpu.py places at
least 2x above the fp32 stand-in's noise and at least 2x below each injected encoder bug.  Depth 2 reaches every
per-block branch of the encoder: block 0's norm1 by the LayerNorm kernel, block 1's by block 0's fused fc2 (or
one-kernel MLP), the last block's fc2 and the final norm.

Each case proves which kernels ran with the launch census of timing mode (`timing` option, `Engine.get_timing`):
`enc_attn` launches are 0 when the fused QKV + attention kernel runs, the `enc_gemm_ln` and `layernorm` counts show
which residual GEMMs carried the LayerNorm that follows them, and the one-kernel MLP replaces the fc1 GEMM.  The routes,
by name in the test ids: the fused residual GEMM + LayerNorm (`fuse_ln` 5: attn.proj, 6: fc2, 7: both, forced at any
batch by bit 2) in each of its modes (MODE 2 column-split CTA pairs, the default at D = 384; MODE 0 single CTAs,
`ln_split` 1 at D = 384 and the default at D = 192; MODE 1 multicast pairs, `ln_cta_group` 2), the one-kernel MLP
(`fuse_mlp`, CTA pairs or single CTAs), both attention implementations (`attn_impl` 0: the fused QKV + attention at
T = 128 and `enc_attention_any_kernel` elsewhere; 1: QKV GEMM + wgmma attention), every image-token count of
token_count_geometries, one image, a batch that fills the persistent GEMM + LayerNorm grid several times in the default
regime, `encode` in chunks, images and weights that are not bf16-representable (the rounding of `im2col_patch_kernel`'s
vector and scalar paths and of the weight conversion), and ViTSTR's class token at T + 1 = 129.

`encode` returns fp32 memory, so it always ends with the unfused LayerNorm; the bf16 memory that a fused final fc2 or
one-kernel MLP writes for `forward` is checked through the decoder (the last test).  Each case prints its statistics
(run with -s to see them)."""
import pytest
import torch

from decoder_reference import BOUNDS as DEC_BOUNDS
from decoder_reference import DecoderReference, budget_stats, excess, format_stats
from encoder_reference import BOUNDS, EncoderReference, sharpen_vitstr
from token_count_geometries import GEOMETRIES, geometry_config

pytestmark = pytest.mark.gpu

WIDTHS = {192: "parseq-tiny", 384: "parseq", 768: "parseq-base-48x160"}
# every launch option a case may set, at its default
DEFAULTS = dict(fuse_ln=3, fuse_mlp=0, ln_split=0, ln_cta_group=0, mlp_cta_group=0, attn_impl=0)
IMAGES = {192: 4, 384: 4, 768: 2}
_MODELS = {}


def _model(D=384, depth=2, T=None, exact=True):
    """(config, state_dict, model) of PARSeq at width D and encoder depth `depth` (T: a token_count_geometries
    geometry); cached, a few at a time."""
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    key = (D, depth, T, exact)
    if key not in _MODELS:
        if len(_MODELS) >= 3:
            _MODELS.clear()
        exp = WIDTHS[D]
        over = dict(geometry_config(T, exp, depth)[1]) if T is not None else dict(enc_depth=depth)
        cfg = make_config(exp, **over)
        sd = init_state_dict(cfg, 31, bf16_exact=exact, sharp=4.0)
        m = create_model(exp, **over)
        m.model.load_state_dict(sd)
        _MODELS[key] = (cfg, sd, m.eval().to("cuda"))
    return _MODELS[key]


def _set(model, opts):
    for k, v in dict(DEFAULTS, **opts).items():
        model.set_engine_option(k, v)


def _census(model, fn):
    """fn()'s result and the launches of each encoder category it issued."""
    eng = model.engine()
    model.set_engine_option("timing", 1)
    try:
        with torch.inference_mode():
            out = fn()
        torch.cuda.synchronize()
        t = eng.get_timing()
    finally:
        model.set_engine_option("timing", 0)
    return out, {k: t[k]["launches"] for k in ("enc_gemm", "enc_attn", "layernorm", "enc_gemm_ln")}


def _expected(depth, proj, fc2, mlp, qkv_attn, chunks=1, final_fused=False):
    """The launches encode_chunk issues per chunk: attn.proj / fc2 with the LayerNorm that follows (`proj`, `fc2`), the
    one-kernel MLP (`mlp`), the fused QKV + attention (`qkv_attn`); `final_fused`: the last block's fc2 (or MLP) also
    produces the final norm, as in `forward`.  `encode` always ends with the LayerNorm kernel (fp32 memory)."""
    gemm, gemm_ln, ln, attn = 1, 0, 0, 0                 # the patch GEMM
    for i in range(depth):
        last = i == depth - 1
        ln += 0 if fc2 and i > 0 else 1                  # norm1: the LayerNorm kernel or the previous block's fc2
        gemm += 1                                        # QKV GEMM or the fused QKV + attention
        attn += 0 if qkv_attn else 1
        gemm, gemm_ln, ln = (gemm, gemm_ln + 1, ln) if proj else (gemm + 1, gemm_ln, ln + 1)
        fused_out = not last or final_fused
        if mlp and fused_out:
            gemm_ln += 1
        else:
            gemm += 1                                    # fc1
            gemm, gemm_ln = (gemm, gemm_ln + 1) if fc2 and fused_out else (gemm + 1, gemm_ln)
    if not final_fused:
        ln += 1
    return {k: v * chunks for k, v in dict(enc_gemm=gemm, enc_attn=attn, layernorm=ln, enc_gemm_ln=gemm_ln).items()}


def _check(name, key, got, ref):
    s = budget_stats(got, ref)
    print(format_stats(f"[{name}] {key}", s))
    assert max(excess(s, key, BOUNDS).values()) <= 1.0, (name, s, BOUNDS[key])


def _encode_case(D, depth, opts, B, *, T=None, exact=True, seed=0):
    """Encodes B images under opts; returns (engine memory, fp64 model memory, census)."""
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(D, depth, T, exact)
    _set(m.model, opts)
    x = synth_images(cfg, B, 40 + seed, bf16_exact=exact).cuda()
    got, census = _census(m.model, lambda: m.model.encode(x))
    ref = EncoderReference(cfg, sd, device="cuda").encode(x)
    assert got.shape == ref.shape == (B, cfg.num_patches, D)
    return got, ref, census


def _flags(D, T, opts, big=False):
    """(proj, fc2, mlp, qkv_attn) as encode_chunk decides them for these options."""
    o = dict(DEFAULTS, **opts)
    fusable = D in (192, 384) and (big or o["fuse_ln"] & 4)
    proj, fc2 = bool(fusable and o["fuse_ln"] & 1), bool(fusable and o["fuse_ln"] & 2)
    return proj, fc2, bool(fc2 and o["fuse_mlp"]), o["attn_impl"] == 0 and T == 128 and D in (192, 384)


# ---- every route at each width, by name -------------------------------------------------------------------------------
def _routes():
    out = []
    modes = {192: [("mode0", {}), ("mode1", dict(ln_cta_group=2))],
             384: [("mode2", {}), ("mode0", dict(ln_split=1)), ("mode1", dict(ln_split=1, ln_cta_group=2))]}
    for D in (192, 384):
        out.append((D, "fuse_ln0", dict(fuse_ln=0)))
        for f in (5, 6, 7):
            for mode, mo in modes[D]:
                out.append((D, f"fuse_ln{f}-{mode}", dict(fuse_ln=f, **mo)))
        for cg in (1, 2):
            out.append((D, f"fuse_mlp-cta_group{cg}", dict(fuse_ln=7, fuse_mlp=1, mlp_cta_group=cg)))
        for f in (0, 7):
            out.append((D, f"attn_wgmma-fuse_ln{f}", dict(fuse_ln=f, attn_impl=1)))
    out += [(768, "fuse_ln0", dict(fuse_ln=0)), (768, "attn_wgmma", dict(fuse_ln=0, attn_impl=1))]
    # depth 1 has no fused fc2 in `encode` (the last block's fc2 precedes the unfused final norm): those routes need 2
    return [(D, depth, name, o) for D, name, o in out for depth in (1, 2)
            if depth == 2 or not name.startswith(("fuse_ln6", "fuse_mlp"))]


ROUTES = _routes()


@pytest.mark.parametrize("case", ROUTES, ids=[f"D{D}-depth{d}-{n}" for D, d, n, _ in ROUTES])
def test_route(case):
    D, depth, name, opts = case
    got, ref, census = _encode_case(D, depth, opts, IMAGES[D])
    proj, fc2, mlp, qkv_attn = _flags(D, 128 if D != 768 else 240, opts)
    assert census == _expected(depth, proj, fc2, mlp, qkv_attn), census
    if name.startswith(("fuse_ln5", "fuse_ln6", "fuse_ln7", "fuse_mlp")):
        assert census["enc_gemm_ln"] > 0
    _check(name, (D, depth), got, ref)


def test_no_fused_variant_at_768():
    """D = 768 has no fused GEMM + LayerNorm: fuse_ln = 7 issues the launches of fuse_ln = 0 and gives the same bits."""
    a, ref, ca = _encode_case(768, 2, dict(fuse_ln=0), 2)
    b, _, cb = _encode_case(768, 2, dict(fuse_ln=7, fuse_mlp=1), 2)
    assert ca == cb and cb["enc_gemm_ln"] == 0
    assert torch.equal(a, b)


@pytest.mark.parametrize("D", sorted(WIDTHS))
def test_images_and_weights_not_bf16_exact(D):
    """Images and weights off the bf16 grid: the patches (im2col_patch_kernel, vector path at pw = 8) and the weights
    (the conversion at load) must be rounded to nearest even, as the model does."""
    got, ref, census = _encode_case(D, 2, dict(fuse_ln=7), IMAGES[D], exact=False, seed=1)
    _check(f"not bf16-exact D{D}", (D, 2), got, ref)


# ---- image-token counts -----------------------------------------------------------------------------------------------
TOKENS = [(T, attn, f) for T in sorted(GEOMETRIES) for attn in (0, 1) for f in (0, 7)]


@pytest.mark.parametrize("case", TOKENS, ids=[f"T{T}-{'attn_wgmma' if a else 'attn_mma'}-fuse_ln{f}" for T, a, f in TOKENS])
def test_image_token_count(case):
    """D = 384 at every geometry of token_count_geometries (ragged last key block, T < 64, ph != pw, the scalar im2col
    path at pw = 4 and 16), with images and weights off the bf16 grid."""
    T, attn, f = case
    opts = dict(fuse_ln=f, attn_impl=attn)
    got, ref, census = _encode_case(384, 2, opts, 3, T=T, exact=False, seed=2)
    assert got.shape[1] == T
    assert census == _expected(2, *_flags(384, T, opts)), census
    _check(f"T{T} attn_impl {attn} fuse_ln {f}", (384, 2), got, ref)


# ---- batches ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [0, 7])
@pytest.mark.parametrize("D", [192, 384])
def test_one_image(D, f):
    got, ref, census = _encode_case(D, 2, dict(fuse_ln=f), 1, seed=3)
    assert census == _expected(2, *_flags(D, 128, dict(fuse_ln=f))), census
    _check(f"one image fuse_ln {f}", (D, 2), got, ref)


def test_default_regime_runs_the_persistent_grid_several_rounds():
    """300 images at T = 128 are 600 tiles of 64 rows: at the default fuse_ln (not forced) and max_batch the residual
    GEMMs run fused, the column-split pairs each walking several tiles."""
    got, ref, census = _encode_case(384, 2, {}, 300, seed=4)
    assert census == _expected(2, *_flags(384, 128, {}, big=True)), census
    assert census["enc_gemm_ln"] == 3
    _check("300 images, default regime", (384, 2), got, ref)


def test_encode_in_chunks():
    """With the `chunk` option below the batch, `encode` runs the encoder once per piece."""
    _, _, m = _model(384, 2)
    m.model.set_engine_option("chunk", 3)
    try:
        got, ref, census = _encode_case(384, 2, dict(fuse_ln=7), 8, seed=5)
    finally:
        m.model.set_engine_option("chunk", 512)
    assert census == _expected(2, *_flags(384, 128, dict(fuse_ln=7)), chunks=3), census
    _check("chunk 3 of 8 images", (384, 2), got, ref)


# ---- ViTSTR -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f", [0, 7])
@pytest.mark.parametrize("attn", [0, 1], ids=["attn_mma", "attn_wgmma"])
def test_vitstr(attn, f):
    """ViTSTR-S at depth 2 (built directly: the system class pins depth 12): the class token and 128 patch tokens,
    forward_features and the tail logits of forward_tokens."""
    from parseq_b200.config import make_config
    from parseq_b200.system import VitstrModel
    from parseq_b200.weights import init_state_dict, synth_images
    cfg = make_config("vitstr", enc_depth=2)
    sd = sharpen_vitstr(init_state_dict(cfg, 32, bf16_exact=(f == 0)), 4.0)
    m = VitstrModel(cfg)
    m.load_state_dict(sd)
    m = m.eval().to("cuda")
    opts = dict(fuse_ln=f, attn_impl=attn)
    _set(m, opts)
    x = synth_images(cfg, 4, 50 + f, bf16_exact=(f == 0)).cuda()
    feats, census = _census(m, lambda: m.forward_features(x))
    with torch.inference_mode():
        logits = m.forward_tokens(x, 25)
    model = EncoderReference(cfg, sd, device="cuda")
    assert feats.shape == (4, cfg.num_patches + 1, cfg.embed_dim) and logits.shape == (4, 26, cfg.num_classes)
    assert census == _expected(2, *_flags(384, 129, opts)), census
    _check(f"ViTSTR features attn_impl {attn} fuse_ln {f}", ("vitstr", 2), feats, model.encode(x))
    _check(f"ViTSTR tail attn_impl {attn} fuse_ln {f}", ("vitstr-tail", 2), logits, model.tail(x, 26))


# ---- the fused final norm, through the decoder ------------------------------------------------------------------------
@pytest.mark.parametrize("mlp", [0, 1], ids=["gemm_ln", "mlp_ln"])
@pytest.mark.parametrize("D", [192, 384])
def test_fused_final_norm_through_the_decoder(D, mlp):
    """`forward` with fuse_ln = 7 takes the decoder's bf16 memory from the last block's fused fc2 (or one-kernel MLP):
    its teacher-free NAR pass, against the fp64 decoder model fed the engine's own fp32 `encode` memory of the same
    images under the same options (x is bit-identical on both routes; only the final LayerNorm's summation order
    differs), stays within the decoder's bounds."""
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(D, 2)
    opts = dict(fuse_ln=7, fuse_mlp=mlp)
    _set(m.model, opts)
    m.model.decode_ar, m.model.refine_iters = False, 0
    x = synth_images(cfg, 6, 60).cuda()
    L = cfg.max_label_length + 1
    with torch.inference_mode():
        mem = m.model.encode(x)
    got, census = _census(m.model, lambda: m.model.forward(m.tokenizer, x, cfg.max_label_length))
    want = _expected(2, True, True, bool(mlp), True, final_fused=True)
    assert {k: census[k] for k in ("enc_gemm", "enc_gemm_ln")} == {k: want[k] for k in ("enc_gemm", "enc_gemm_ln")}
    ref = DecoderReference(cfg, sd, device="cuda").nar(mem, L)
    assert got.shape == ref.shape == (6, L, cfg.num_classes)
    s = budget_stats(got, ref)
    print(format_stats(f"[fused final norm {'mlp_ln' if mlp else 'gemm_ln'}] D {D}", s))
    assert max(excess(s, (D, 1), DEC_BOUNDS).values()) <= 1.0, (s, DEC_BOUNDS[(D, 1)])
