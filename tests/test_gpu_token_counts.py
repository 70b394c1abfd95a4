"""GPU: the PARSeq decoder at every image-token-count regime the kernels distinguish.  The cluster AR kernel streams an
image's cross K/V in 64-row boxes (T <= 64) or 128-row key blocks; the other decoder paths mask keys >= T in their own
ways; the patch GEMM's K is 3 * ph * pw.  Each geometry is checked against the live fp32 ParseqOracle (encoder depth 2,
sharp attention weights, so that a leaked or dropped key moves the logits far outside the tolerance), across the three
AR implementations, on the uint8 input path and through `model.decode` with a padding mask."""
import pytest
import torch

from token_count_geometries import GEOMETRIES, geometry_config

pytestmark = pytest.mark.gpu

TOL_FP32_MAX = 2.0e-2          # the bounds of test_gpu_parity.py
TOL_FP32_MEAN = 3.0e-3
TAU = 2.0e-2

# (T, experiment): D = 384 at every T, D = 192 (parseq-tiny) at 49 and 130, D = 768 at 65
CASES = [(T, "parseq") for T in sorted(GEOMETRIES)] + [(49, "parseq-tiny"), (130, "parseq-tiny"),
                                                       (65, "parseq-base-48x160")]


def _ids(c):
    return f"T{c[0]}-{c[1]}"


def _model(T, experiment, seed=13):
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg, over = geometry_config(T, experiment)
    sd = init_state_dict(cfg, seed, sharp=4.0)
    m = create_model(experiment, **over)
    m.model.load_state_dict(sd)
    return cfg, sd, m.eval().to("cuda")


@pytest.mark.parametrize("T,experiment", CASES, ids=[_ids(c) for c in CASES])
@pytest.mark.parametrize("ar,ri", [(True, 1), (False, 2)], ids=["ar1", "nar2"])
def test_teacher_forced_vs_live_fp32_oracle(T, experiment, ar, ri):
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(T, experiment)
    m.model.decode_ar, m.model.refine_iters = ar, ri
    x = synth_images(cfg, 6, 40 + T)
    o = ParseqOracle(cfg, sd, "fp32").forward(x, 25, ar, ri)
    forced = o.ar_ids.int() if o.ar_ids is not None else None
    forced_refine = torch.stack([c.int() for c in o.refine_ctx]) if o.refine_ctx else None
    with torch.inference_mode():
        lf = m.model.forward(m.tokenizer, x.cuda(), 25, forced_ids=forced, forced_refine=forced_refine).cpu()
    # as for the sharp goldens of test_gpu_parity.py: operand rounding is amplified by the sharp attention (D = 768 most),
    # so the bound is 1.5x the deviation of the rounding-point model (oracle, precision "bf16") from the same fp32
    # reference on the same trajectory, never tighter than the plain tolerance
    ob = ParseqOracle(cfg, sd, "bf16").forward(x, 25, ar, ri, forced_ids=o.ar_ids, forced_refine=o.refine_ctx or None)
    model_err = (ob.logits - o.logits).abs()
    tol_max = max(TOL_FP32_MAX, 1.5 * model_err.max().item())
    tol_mean = max(TOL_FP32_MEAN, 1.5 * model_err.mean().item())
    tau = max(TAU, tol_max)
    err = (lf - o.logits).abs()
    assert err.max().item() <= tol_max and err.mean().item() <= tol_mean, (err.max().item(), err.mean().item(), tol_max)
    top2 = o.logits.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > tau
    assert bool((lf.argmax(-1) == o.logits.argmax(-1))[clear].all())
    assert int(clear.sum()) > clear.numel() // 4


@pytest.mark.parametrize("T,experiment", CASES, ids=[_ids(c) for c in CASES])
def test_ar_loop_implementations_agree(T, experiment):
    """As test_gpu_parity.test_ar_loop_implementations_agree, at this T, for the instantiations a batch size selects:
    the head-split cluster kernel at B = 1, one m16 row tile at a small batch, two row tiles above 16 x the co-resident
    clusters (not for D = 768, which has no two-tile variant and runs the small batches only), each with clusters of 8
    and of 6."""
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(T, experiment)
    m.model.decode_ar, m.model.refine_iters = True, 0
    eng = m.model.engine()
    for B in ((1, 19) if cfg.embed_dim == 768 else (1, 19, 300)):
        x = synth_images(cfg, B, 50 + B).cuda()
        g = torch.Generator().manual_seed(B)
        forced = torch.randint(0, cfg.num_classes, (B, 26), generator=g, dtype=torch.int32)
        forced[:, 0] = m.bos_id
        outs, reached = {}, {}
        with torch.inference_mode():
            for impl, cs in ((2, 8), (2, 6), (1, 0), (0, 0)):
                m.model.set_engine_option("ar_kernel", impl)
                if cs:
                    m.model.set_engine_option("ar_cluster_size", cs)
                outs[(impl, cs)] = m.model.forward(m.tokenizer, x, 25, forced_ids=forced).cpu()
                if impl == 2:
                    reached[cs] = (eng.debug_int("ar_last_cluster_size"), eng.debug_int("ar_last_per"))
        assert reached[8][0] == 8 and reached[6][0] == 6, reached
        if B == 1:
            assert reached[8][1] == 1                                         # head-split regime
        elif B == 300:
            assert reached[8][1] > 16 or reached[6][1] > 16, reached         # two m16 row tiles
        ref = outs[(2, 8)]
        for key, out in outs.items():
            d = (ref - out).abs()
            assert d.max().item() <= 8e-3 and d.mean().item() <= 8e-4, (B, key, d.max().item(), d.mean().item())
            top2 = out.topk(2, dim=-1).values
            clear = (top2[..., 0] - top2[..., 1]) > 1e-2
            assert bool((ref.argmax(-1) == out.argmax(-1))[clear].all())


@pytest.mark.parametrize("T,experiment", CASES, ids=[_ids(c) for c in CASES])
def test_uint8_input_path_is_bit_identical_to_float_path(T, experiment):
    cfg, sd, m = _model(T, experiment)
    H, W = cfg.img_size
    g = torch.Generator().manual_seed(T)
    u8 = torch.randint(0, 256, (5, H, W, 3), dtype=torch.uint8, generator=g)
    xf = (u8.permute(0, 3, 1, 2).to(torch.float32).div(255) - 0.5) / 0.5          # ToTensor, Normalize(0.5, 0.5)
    with torch.inference_mode():
        lf = m(xf.cuda())
        lu = m(u8.cuda())
    assert torch.equal(lf, lu)


@pytest.mark.parametrize("T,experiment", [(49, "parseq"), (130, "parseq-tiny")], ids=["T49-parseq", "T130-parseq-tiny"])
def test_decode_with_padding_mask(T, experiment):
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(T, experiment)
    o = ParseqOracle(cfg, sd, "fp32")
    B, L = 3, 26
    g = torch.Generator().manual_seed(T)
    memory = o.encode(synth_images(cfg, B, T))
    tgt = torch.randint(1, cfg.num_classes, (B, L), generator=g)
    tgt[:, 0] = m.bos_id
    qmask = torch.zeros((L, L), dtype=torch.bool)
    qmask[torch.arange(L - 1), torch.arange(1, L)] = True
    pmask = torch.rand((B, L), generator=g) < 0.3
    pmask[:, 0] = False
    ref = o._decode(tgt, memory, o.p["pos_queries"][:, :L].expand(B, -1, -1), qmask, pmask)
    with torch.inference_mode():
        out = m.model.decode(tgt.cuda(), memory.cuda(), tgt_query_mask=qmask.cuda(), tgt_padding_mask=pmask.cuda())
        logits = m.model.head(out).cpu()
    err = (logits - ref).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN, (err.max().item(), err.mean().item())
