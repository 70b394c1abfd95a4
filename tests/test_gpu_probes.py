"""GPU: the engine on the probe models of tests/probe_models.py, against their fp64 model, route by route.

Each probe makes one detail of the arithmetic (an extra or a missing key, P rounded before or after the division by the
row sum, the GELU form, the LayerNorm eps, the cross query's low bits, the rounding of patches and weights) move the
output by 7e-3 to 26 while a correct engine agrees with the fp64 model to ~1e-6, so the tolerance of 1e-4 holds the
engine to the right arithmetic where the statistical budgets of test_gpu_encoder_isolated.py and
test_gpu_decoder_isolated.py cannot (tests/test_probe_separation_cpu.py shows every covered bug 10x over it).

Encoder probes run under every route of test_gpu_encoder_isolated.ROUTES, proven by the same launch census, and ViTSTR's
under both attention implementations with and without the fused GEMM + LayerNorm.  Decoder probes run on the engine's
own memory (the +-1 pattern, checked exactly) through every cluster-kernel instantiation of
test_gpu_decoder_isolated.py (each proven by the full reach tuple: path, MT, cluster size, head split, class-sliced head,
ids pitch), the grid-barrier kernel, the chain, NAR, refinement and depth 2.  The cross-attention probe also runs at
T = 32, 65, 130 and 240 image tokens, where key T lies inside a zero-filled K/V box (an extra key would be read), and
at T = 256, where the last key ends the last box.  Each case prints its error (run with -s to see it)."""
import pytest
import torch

import probe_models as pm
from test_gpu_encoder_isolated import ROUTES as ENC_ROUTES
from test_gpu_encoder_isolated import _census, _expected, _flags, _set
from test_gpu_decoder_isolated import AR_CASES as DEC_AR_CASES
from test_gpu_decoder_isolated import ROUTES as DEC_AR_ROUTES

pytestmark = pytest.mark.gpu

_MODELS = {}


def _engine(p):
    """The engine loaded with the probe's weights; cached, a few at a time."""
    from parseq_b200.factory import create_model
    from parseq_b200.system import VitstrModel
    if p.name not in _MODELS:
        if len(_MODELS) >= 3:
            _MODELS.clear()
        if p.cfg.arch == "vitstr":
            m = VitstrModel(p.cfg)
            m.load_state_dict(p.sd)
            m = m.eval().to("cuda")
        else:
            over = dict(p.over) if p.over else dict(enc_depth=p.cfg.enc_depth)
            over["dec_depth"] = p.cfg.dec_depth
            m = create_model(pm.EXPERIMENT[p.key[0]], **over)
            m.model.load_state_dict(p.sd)
            m = m.eval().to("cuda")
            m.model.set_engine_option("max_batch", 64)
        _MODELS[p.name] = m
    return _MODELS[p.name]


_PROBES = {}


def _probe(fn, *args):
    while args and args[-1] is None:
        args = args[:-1]
    k = (fn.__name__, args)
    if k not in _PROBES:
        _PROBES[k] = fn(*args)
    return _PROBES[k]


def _check(p, what, got, ref):
    e = (got.double() - ref.double()).abs().max().item()
    print(f"[{p.name} {what}] max |engine - model| {e:.2e}  tolerance {p.tol:.0e}")
    assert torch.isfinite(got).all()
    assert e <= p.tol, (p.name, what, e)


# ---- the encoder --------------------------------------------------------------------------------------------------
ENC_KINDS = [pm.enc_attention, pm.enc_gelu, pm.enc_ln_eps]
ENC_CASES = [(fn, D, depth, name, opts) for fn in ENC_KINDS for D, depth, name, opts in ENC_ROUTES]


@pytest.mark.parametrize("case", ENC_CASES, ids=[f"{c[0].__name__}-D{c[1]}-depth{c[2]}-{c[3]}" for c in ENC_CASES])
def test_encoder_probe(case):
    fn, D, depth, name, opts = case
    p = _probe(fn, (D, depth))
    m = _engine(p)
    _set(m.model, opts)
    x = p.images.cuda()
    got, census = _census(m.model, lambda: m.model.encode(x))
    assert census == _expected(depth, *_flags(D, p.cfg.num_patches, opts)), census
    _check(p, name, got, p.expected(device="cuda"))


VIT_KINDS = [pm.enc_attention, pm.enc_gelu, pm.enc_ln_eps, pm.vitstr_rounding]
VIT_CASES = [(fn, key, attn, f) for fn in VIT_KINDS for key in (("vitstr", 2), ("vitstr-tail", 2))
             for attn in (0, 1) for f in (0, 7)]


@pytest.mark.parametrize("case", VIT_CASES,
                         ids=[f"{c[0].__name__}-{c[1][0]}-attn_impl{c[2]}-fuse_ln{c[3]}" for c in VIT_CASES])
def test_vitstr_probe(case):
    fn, key, attn, f = case
    p = _probe(fn, key)
    m = _engine(p)
    opts = dict(fuse_ln=f, attn_impl=attn)
    _set(m, opts)
    x = p.images.cuda()
    if key[0] == "vitstr":
        got, census = _census(m, lambda: m.forward_features(x))
        assert census == _expected(2, *_flags(384, 129, opts)), census
    else:
        with torch.inference_mode():
            got = m.forward_tokens(x, pm.L_TAIL - 1)
    _check(p, f"attn_impl {attn} fuse_ln {f}", got, p.expected(device="cuda"))


# ---- the decoder --------------------------------------------------------------------------------------------------
# every cluster-kernel instantiation of test_gpu_decoder_isolated.py, by (MT, CS, head split), the class-sliced head
# (195 classes) and the ids pitch (32: L = 26, 64: L = 64), with its batch and options; then the other AR routes and
# passes
AR_CASES = [(fn, D, r, wide, pitch) for fn in (pm.dec_cross, pm.dec_ln_eps) for D, r, wide, pitch in DEC_AR_CASES]
# name -> (batch, engine options, the ar_last_path reached or None, widths)
PASSES = {
    "grid-barrier": (6, (("ar_kernel", 1),), 1, (192, 384)),
    "chain": (6, (("ar_kernel", 0),), 0, (192, 384, 768)),
    "nar": (6, (), None, (192, 384, 768)),
    "refine": (6, (), None, (192, 384, 768)),
}
DEC_CASES = [(fn, (D, 1), None, r) for fn in (pm.dec_cross, pm.dec_ln_eps) for D in (192, 384, 768)
             for r, v in PASSES.items() if D in v[3]]
DEC_CASES += [(fn, (384, 2), None, r) for fn in (pm.dec_cross, pm.dec_ln_eps) for r in ("chain", "nar", "refine")]
DEC_CASES += [(pm.dec_cross, (384, 1), T, r) for T in pm.CROSS_T for r in ("cluster", "chain")]
PASSES["cluster"] = (2, (), 2, (384,))


def _repeat(t, B):
    return t.repeat((B + t.shape[0] - 1) // t.shape[0], *([1] * (t.dim() - 1)))[:B]


def _run(p, B, opts):
    """Runs the probe's batch (repeated to B images) under opts; returns (engine logits, fp64 model logits)."""
    m = _engine(p)
    for k, v in (("fuse_ln", 0), ("ar_kernel", 2), ("ar_cluster_size", 0), ("ar_clusters", 0)) + tuple(opts):
        m.model.set_engine_option(k, v)
    ar, refine = m.model.decode_ar, m.model.refine_iters
    x = _repeat(p.images, B).cuda()
    forced = _repeat(p.forced, B) if ar else None
    ctx = _repeat(p.context, B)
    with torch.inference_mode():
        mem = m.model.encode(x)
        got = m.model.forward(m.tokenizer, x, p.cfg.max_label_length, forced_ids=forced,
                              forced_refine=ctx[None] if refine else None)
    memr = mem.to(torch.bfloat16).float()
    assert torch.equal(memr.cpu(), _repeat(p.memory(), B)), "the probe's memory is not the +-1 pattern"
    cluster = bool(ar and not refine and m.model.engine().debug_int("ar_last_path") == 2)
    q = pm.Probe(**{**p.__dict__, "images": x.cpu(), "forced": forced, "context": ctx})
    ref = q.expected(device="cuda", memory=memr, cluster=cluster, pass_="refine" if refine else "ar" if ar else "nar")
    return got, ref


def _ar_id(c):
    fn, D, (mt, cs, hs), wide, pitch = c
    return f"{fn.__name__}-D{D}-mt{mt}-cs{cs}-hs{hs}-{'wide' if wide else 'c95'}-idp{pitch}"


@pytest.mark.parametrize("case", AR_CASES, ids=[_ar_id(c) for c in AR_CASES])
def test_decoder_probe_cluster_instantiation(case):
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


@pytest.mark.parametrize("case", DEC_CASES, ids=[f"{c[0].__name__}-D{c[1][0]}-depth{c[1][1]}"
                                                 f"{'-T%d' % c[2] if c[2] else ''}-{c[3]}" for c in DEC_CASES])
def test_decoder_probe(case):
    fn, key, T, route = case
    p = _probe(fn, key, T)
    B, opts, path, _ = PASSES[route]
    m = _engine(p)
    m.model.decode_ar, m.model.refine_iters = route not in ("nar", "refine"), int(route == "refine")
    got, ref = _run(p, B, opts)
    if path is not None:
        assert m.model.engine().debug_int("ar_last_path") == path
    _check(p, route, got, ref)
