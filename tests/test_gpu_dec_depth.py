"""GPU: PARSeq decoders of depth 2 and 3.  The engine runs the content stream of layers 0..N-2 and the query stream of
every layer on the chain of separate kernels (the cluster AR kernel covers depth 1 only).  Checked against the reference
goldens (tests/golden/depth), against the live depth-N oracle, and for the properties that need no reference: rows do not
depend on the batch, graph replay equals eager, a NaN crop stays in its own image."""
import glob
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "depth")
TOL_FP32_MAX = 2.0e-2          # the bounds of test_gpu_parity.py
TOL_FP32_MEAN = 3.0e-3
TAU = 2.0e-2
FORWARD_CASES = sorted(p for p in glob.glob(os.path.join(GOLDEN, "d*_*.pt"))
                       if "refine_" not in p and "decode_" not in p and "state_dict" not in p)


def _model(experiment, depth, mll=25, seed=0, n_extra=0, sharp=0.0, **kw):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config_long(experiment, mll, n_extra, dec_depth=depth)
    sd = init_state_dict(cfg, seed, sharp=sharp)
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=mll, dec_depth=depth, **kw)
    m.model.load_state_dict(sd)
    return cfg, sd, m.eval().to("cuda")


def _blob_model(blob, **kw):
    return _model(blob["experiment"], blob["dec_depth"], blob["max_label_length"], blob["weight_seed"], blob["n_extra"],
                  blob.get("sharp", 0.0), decode_ar=blob["decode_ar"], refine_iters=blob["refine_iters"], **kw)


def _forced(blob, L):
    forced = forced_refine = None
    if blob.get("ar_ids") is not None:
        forced = torch.zeros((blob["batch"], L), dtype=torch.int32)
        forced[:, : blob["ar_ids"].shape[1]] = blob["ar_ids"]
    if blob["refine_ctx"]:
        forced_refine = torch.zeros((len(blob["refine_ctx"]), blob["batch"], L), dtype=torch.int32)
        for r, c in enumerate(blob["refine_ctx"]):
            forced_refine[r, :, : c.shape[1]] = c
    return forced, forced_refine


def _run(m, x, max_length=None, forced=None, forced_refine=None):
    with torch.inference_mode():
        logits, ids = m.model.forward(m.tokenizer, x.cuda(), max_length, return_ids=True,
                                      forced_ids=None if forced is None else forced.cuda(),
                                      forced_refine=None if forced_refine is None else forced_refine.cuda())
    torch.cuda.synchronize()
    return logits.cpu(), ids.cpu()


def _close(a, b):
    err = (a - b).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN, (err.max().item(), err.mean().item())


@pytest.mark.parametrize("path", FORWARD_CASES, ids=lambda p: os.path.basename(p)[:-3])
def test_teacher_forced_parity_with_reference_golden(path):
    """AR + refine, NAR + refine, AR only (early exit), L = 64, 3001 classes, max_length < L: the engine driven along the
    reference's own id trajectory reproduces its logits, and every clear decision."""
    from parseq_b200.weights import synth_images
    blob = torch.load(path, weights_only=False)
    cfg, sd, m = _blob_model(blob)
    x = synth_images(cfg, blob["batch"], blob["image_seed"])
    L = m.model.engine().num_steps(blob["max_length"])
    forced, forced_refine = _forced(blob, L)
    logits, ids = _run(m, x, blob["max_length"], forced, forced_refine)
    assert m.model.engine().debug_int("ar_last_cluster_size") == 0       # the cluster kernel never ran
    ref = blob["logits"]
    assert logits.shape == ref.shape
    _close(logits, ref)
    top2 = ref.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > TAU
    assert torch.equal(ids.long()[clear], ref.argmax(-1)[clear])


def test_refine_with_eos_in_both_key_groups_sharp_weights():
    """Cloze refinement at L = 64 on sharp weights, first EOS in either 32-key group: the content stream runs under the
    cloze + first-EOS mask.  Bound: 1.5x the bf16 rounding-point model's own distance to the reference."""
    from dec_depth_oracle import DepthOracle
    from make_golden_long import cloze_masks
    from parseq_b200.weights import synth_images
    blob = torch.load(os.path.join(GOLDEN, "d2_eos_s_refine_b4.pt"), weights_only=False)
    cfg, sd, m = _model(blob["experiment"], 2, 63, blob["weight_seed"], sharp=blob["sharp"], decode_ar=False, refine_iters=1)
    x = synth_images(cfg, blob["batch"], blob["image_seed"])
    ctx = blob["refine_ctx"][0]
    logits, _ = _run(m, x, 63, None, ctx[None])
    ref = blob["logits"]
    o = DepthOracle(cfg, sd, "bf16")
    B, L = ctx.shape
    qmask, pmask = cloze_masks(ctx.long())
    model = o._decode(ctx.long(), o.r(o.encode(x)), o.p["pos_queries"][:, :L].expand(B, -1, -1), qmask, pmask, qmask).float()
    bound = max(TOL_FP32_MAX, 1.5 * (model - ref).abs().max().item())
    assert (logits - ref).abs().max().item() <= bound


@pytest.mark.parametrize("depth,experiment", [(2, "parseq-tiny"), (3, "parseq")])
def test_free_running_ids_match_fp32_oracle(depth, experiment):
    """Free-running AR decoding (no teacher forcing): up to each image's first decision whose fp32 margin is <= tau, the
    engine's contexts equal the oracle's, so those ids agree and the logits up to that step are within tolerance."""
    from dec_depth_oracle import DepthOracle
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(experiment, depth, seed=11, decode_ar=True, refine_iters=0)
    x = synth_images(cfg, 4, 11)
    logits, ids = _run(m, x)
    o = DepthOracle(cfg, sd, "fp32").forward(x, None, True, 0)
    top2 = o.ar_logits.topk(2, dim=-1).values
    margin = top2[..., 0] - top2[..., 1]
    S = min(ids.shape[1], o.ids.shape[1])
    checked = 0
    for b in range(x.shape[0]):
        low = (margin[b, :S] <= TAU).nonzero()
        k = int(low[0]) if len(low) else S
        assert torch.equal(ids[b, :k].long(), o.ids[b, :k])
        _close(logits[b, : min(k + 1, S)], o.logits[b, : min(k + 1, S)])
        checked += k
    assert checked > 0


def test_no_cluster_kernel_and_grid_barrier_kernel_rejected():
    from parseq_b200.engine import EngineError
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny", 2, decode_ar=True, refine_iters=1)
    eng = m.model.engine()
    with pytest.raises(EngineError, match="ar_kernel"):
        eng.set_option("ar_kernel", 1)
    eng.set_option("timing", 1)
    _run(m, synth_images(cfg, 2, 0))
    t = eng.get_timing()
    eng.set_option("timing", 0)
    assert t["dec_ar"]["launches"] == 0 and t["dec_attn"]["launches"] > 0


def test_depth_below_one_is_rejected():
    from parseq_b200.config import make_config
    from parseq_b200.engine import Engine, EngineError
    with pytest.raises(EngineError, match="dec_depth"):
        Engine(make_config("parseq-tiny", dec_depth=0), 0)


def test_rows_do_not_depend_on_the_batch_and_graph_equals_eager():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 2, seed=4, decode_ar=True, refine_iters=1)
    x = synth_images(cfg, 6, 4)
    full, ids_full = _run(m, x)
    for lo, hi in ((0, 1), (2, 5)):
        part, ids_part = _run(m, x[lo:hi])
        assert torch.equal(part, full[lo:hi]) and torch.equal(ids_part, ids_full[lo:hi])
    m.model.set_engine_option("use_graph", 0)
    eager, ids_eager = _run(m, x)
    m.model.set_engine_option("use_graph", 1)
    assert torch.equal(eager, full) and torch.equal(ids_eager, ids_full)


def test_batch_above_max_batch_equals_its_halves_and_dec_chunks():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny", 3, seed=5, decode_ar=True, refine_iters=2)
    x = synth_images(cfg, 8, 5)
    whole, _ = _run(m, x)
    m.model.set_engine_option("max_batch", 4)
    m.model.set_engine_option("dec_chunk", 2)
    split, _ = _run(m, x)
    a, _ = _run(m, x[:4])
    assert torch.equal(split, whole) and torch.equal(a, whole[:4])


def test_nar_and_max_length_below_L():
    from dec_depth_oracle import DepthOracle
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny", 2, seed=6, decode_ar=False, refine_iters=2)
    x = synth_images(cfg, 3, 6)
    logits, _ = _run(m, x, 7)
    assert logits.shape == (3, 8, 95)
    o = DepthOracle(cfg, sd, "fp32").forward(x, 7, False, 2)
    sure = o.min_margin > TAU
    _close(logits[sure], o.logits[sure])


def test_nan_crop_leaves_other_images_bit_identical():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny", 2, seed=7, decode_ar=True, refine_iters=1)
    x = synth_images(cfg, 3, 7)
    clean, _ = _run(m, x)
    x[1, :, 3, 5] = float("nan")
    dirty, _ = _run(m, x)
    assert torch.equal(dirty[0], clean[0]) and torch.equal(dirty[2], clean[2])


def test_decode_content_mask_matches_reference_golden():
    """PARSeq.decode with custom queries, a query mask, a padding mask and tgt_mask: the content mask is honoured, and the
    fully masked content row of image 2 turns that image's outputs into NaN as the reference's do."""
    blob = torch.load(os.path.join(GOLDEN, "d2_decode_ti_b3.pt"), weights_only=False)
    cfg, sd, m = _model(blob["experiment"], 2, 25, blob["weight_seed"])
    dev = "cuda"
    args = dict(tgt_padding_mask=blob["padding_mask"].to(dev), tgt_query=blob["query"].to(dev),
                tgt_query_mask=blob["query_mask"].to(dev))
    with torch.inference_mode():
        out = m.model.decode(blob["ids"].to(dev), blob["memory"].to(dev), blob["content_mask"].to(dev), **args).cpu()
        free = m.model.decode(blob["ids"].to(dev), blob["memory"].to(dev), None, **args).cpu()
    ref = blob["out"]
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(out), nan)
    _close(out[~nan], ref[~nan])
    assert not torch.isnan(free).any()
    _close(free, blob["out_no_content_mask"])


def test_u8_path_equals_float_path():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny", 2, seed=8, decode_ar=True, refine_iters=1)
    eng = m.model.engine()
    u8 = (synth_images(cfg, 2, 8, bf16_exact=False) * 127.5 + 127.5).round().clamp(0, 255).to(torch.uint8)
    hwc = u8.permute(0, 2, 3, 1).contiguous().cuda()
    x = (u8.float() / 255.0 - 0.5) / 0.5
    ref, _ = _run(m, x)
    L = eng.num_steps(None)
    logits = torch.empty((2, L, cfg.num_classes), device="cuda")
    ids = torch.empty((2, L), dtype=torch.int32, device="cuda")
    steps = torch.empty((1,), dtype=torch.int32, device="cuda")
    eng.forward_u8(hwc.data_ptr(), 2, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(),
                   torch.cuda.current_stream().cuda_stream, None, True, 1)
    torch.cuda.synchronize()
    assert torch.equal(logits.cpu(), ref)
