"""GPU: per-image character allowlists (parseq_forward_args.class_mask; PARSeq / ViTSTR `forward(..., allowlist=...)`).

The engine must behave as the reference whose head returns -inf for every class an image does not allow
(tests/allowlist_oracle.py): checked against goldens of the reference's own modules with the wrapped head
(tests/golden/allowlist) on every AR implementation, and for the properties that need no reference - an all-ones mask is
a NULL mask bit for bit, images of a batch do not affect each other, graph replay equals eager, host equals device
entry points, raw crops equal their preprocessed stack, super-chunks equal their halves, a NaN crop stays EOS."""
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "allowlist")
TOL_FP32_MAX = 2.0e-2          # the bounds of test_gpu_parity.py
TOL_FP32_MEAN = 3.0e-3
TAU = 2.0e-2
DIGITS = "0123456789"
PARSEQ_CASES = sorted(p for p in glob.glob(os.path.join(GOLDEN, "al_*.pt")) if "vitstr" not in os.path.basename(p))


def _model(experiment, mll=25, seed=0, n_extra=0, dec_depth=1, **kw):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    extra = {} if experiment == "vitstr" else {"dec_depth": dec_depth}
    cfg = make_config_long(experiment, mll, n_extra, **extra)
    sd = init_state_dict(cfg, seed)
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=mll, **extra, **kw)
    (m if experiment == "vitstr" else m.model).load_state_dict(sd)
    return cfg, sd, m.eval().to("cuda")


def _run(m, x, mask, max_length=None):
    """(logits, ids) of one call; PARSeq logits are cut to the S steps the batch ran when refine_iters == 0."""
    with torch.inference_mode():
        if hasattr(m.model, "forward_tokens"):
            return m.model.forward_tokens(x, max_length, return_ids=True, class_mask=mask)
        return m.model.forward(m.tokenizer, x, max_length, return_ids=True, class_mask=mask)


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _check_masked(logits, allowed):
    """Disallowed classes hold exactly -inf."""
    assert bool(torch.isneginf(logits)[~allowed[:, None, :].expand_as(logits)].all())


# (name, engine options): every AR implementation the golden's model can run
AR_IMPLS = {
    "cluster": {"ar_kernel": 2, "ar_clusters": 1},      # one cluster: the redundant (or WIDE) head on whole images
    "cluster_hs": {"ar_kernel": 2},                     # small batches: one (image, head pair) per CTA
    "grid": {"ar_kernel": 1},
    "chain": {"ar_kernel": 0},
}


def _applies(blob, impl, C):
    if impl == "grid":
        return C <= 128 and blob["max_label_length"] <= 31 and blob["dec_depth"] == 1
    if impl.startswith("cluster"):
        return blob["dec_depth"] == 1 and (C <= 96 or C > 128)
    return True


@pytest.mark.parametrize("impl", list(AR_IMPLS))
@pytest.mark.parametrize("path", PARSEQ_CASES, ids=lambda p: os.path.basename(p)[:-3])
def test_ids_and_logits_vs_reference_golden(path, impl):
    from allowlist_oracle import allowed_from_strings
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(path, weights_only=False)
    cfg, sd, m = _model(blob["experiment"], blob["max_label_length"], blob["weight_seed"], blob["n_extra"],
                        blob["dec_depth"], decode_ar=blob["decode_ar"], refine_iters=blob["refine_iters"])
    assert state_dict_digest(sd) == blob["sd_digest"]
    if not _applies(blob, impl, cfg.num_classes):
        pytest.skip(f"{impl} does not run this model's AR loop")
    for k, v in AR_IMPLS[impl].items():
        m.model.set_engine_option(k, v)
    B = blob["batch"]
    x = synth_images(cfg, B, blob["image_seed"]).cuda()
    mask = m.allowlist_mask(blob["allowlist"], B)
    logits, ids = _run(m, x, mask, blob["max_length"])
    logits, ids = logits.cpu(), ids.cpu()
    if blob["decode_ar"] and impl.startswith("cluster"):
        eng = m.model.engine()
        assert eng.debug_int("ar_last_wide") == int(cfg.num_classes > 128)
        if impl == "cluster_hs" and B <= 15:
            assert eng.debug_int("ar_last_head_split") == 1
        if impl == "cluster":
            assert eng.debug_int("ar_last_head_split") == 0
    allowed = allowed_from_strings(m.tokenizer, blob["allowlist"], cfg.num_classes)
    ref, ref_ids = blob["logits"], blob["ids"].long()
    clear = blob["min_margin_fp64"] > TAU
    assert int(clear.sum()) >= 1
    if bool(clear.all()):
        assert logits.shape == ref.shape                # S of refine_iters == 0 from the masked ids
    S = min(logits.shape[1], ref.shape[1])
    _check_masked(logits, allowed)
    assert torch.equal(ids.long(), logits.argmax(-1))
    assert torch.equal(ids[clear, :S].long(), ref_ids[clear, :S])
    fin = torch.isfinite(ref[clear, :S])
    err = (logits[clear, :S] - ref[clear, :S])[fin].abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN, (err.max().item(), err.mean().item())
    assert torch.equal(torch.isneginf(logits[clear, :S]), torch.isneginf(ref[clear, :S]))
    labels, _ = m.postprocess(logits.cuda())
    for lab, a in zip(labels, blob["allowlist"]):
        assert a is None or set(lab) <= set(a), (lab, a)


def test_vitstr_vs_reference_golden():
    from allowlist_oracle import allowed_from_strings
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(os.path.join(GOLDEN, "al_vitstr_s_b4.pt"), weights_only=False)
    cfg, sd, m = _model("vitstr", blob["max_label_length"], blob["weight_seed"])
    assert state_dict_digest(sd) == blob["sd_digest"]
    x = synth_images(cfg, blob["batch"], blob["image_seed"]).cuda()
    logits, ids = _run(m, x, m.allowlist_mask(blob["allowlist"], blob["batch"]), blob["max_length"])
    logits, ids = logits.cpu(), ids.cpu()
    ref = blob["logits"]
    allowed = allowed_from_strings(m.tokenizer, blob["allowlist"], cfg.num_classes)
    _check_masked(logits, allowed)
    fin = torch.isfinite(ref)
    err = (logits - ref)[fin].abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN
    top2 = ref.topk(2, dim=-1).values                  # no feedback in ViTSTR: every clear position on its own
    clear = (top2[..., 0] - top2[..., 1]) > TAU
    assert bool((ids.long() == ref.argmax(-1))[clear].all())
    labels, _ = m.postprocess(logits.cuda())
    for lab, a in zip(labels, blob["allowlist"]):
        assert a is None or set(lab) <= set(a)


# (experiment, extra characters, engine options, decode_ar, refine_iters): every AR path and the NAR pass
ONES_PATHS = {
    "cluster": ("parseq", 0, {}, True, 1),
    "cluster_ar0": ("parseq", 0, {}, True, 0),
    "grid": ("parseq", 0, {"ar_kernel": 1}, True, 1),
    "chain": ("parseq", 0, {"ar_kernel": 0}, True, 0),
    "nar": ("parseq", 0, {}, False, 2),
    "wide": ("parseq-tiny", 2906, {}, True, 1),
    "wide_chain": ("parseq-tiny", 2906, {"ar_kernel": 0}, True, 1),
    "vitstr": ("vitstr", 0, {}, None, None),
}


@pytest.mark.parametrize("B", [1, 7, 512])
@pytest.mark.parametrize("path", list(ONES_PATHS))
def test_all_ones_mask_is_bit_identical_to_no_mask(path, B):
    from make_golden_long import charset
    from parseq_b200.weights import synth_images
    exp, n_extra, opts, ar, ri = ONES_PATHS[path]
    if n_extra and B == 512:
        pytest.skip("the 3001-class head at bs 512 repeats bs 7 at 70x the logits")
    kw = {} if exp == "vitstr" else {"decode_ar": ar, "refine_iters": ri}
    cfg, sd, m = _model(exp, 25, 11, n_extra, **kw)
    for k, v in opts.items():
        m.model.set_engine_option(k, v)
    x = synth_images(cfg, B, 140).cuda()
    base, base_ids = _run(m, x, None)
    ones, ones_ids = _run(m, x, m.allowlist_mask(charset(n_extra), B))
    assert _same(base, ones) and torch.equal(base_ids, ones_ids)


@pytest.mark.parametrize("path", ["cluster", "chain", "nar", "vitstr"])
def test_unmasked_images_of_a_masked_batch_are_unchanged(path):
    from parseq_b200.weights import synth_images
    exp, n_extra, opts, ar, ri = ONES_PATHS[path]
    kw = {} if exp == "vitstr" else {"decode_ar": ar, "refine_iters": ri}
    cfg, sd, m = _model(exp, 25, 12, n_extra, **kw)
    for k, v in opts.items():
        m.model.set_engine_option(k, v)
    x = synth_images(cfg, 512, 141).cuda()
    base, base_ids = _run(m, x, None, 25)
    allow = [DIGITS if b % 2 else None for b in range(512)]
    got, got_ids = _run(m, x, m.allowlist_mask(allow, 512), 25)
    assert _same(got[0::2], base[0::2]) and torch.equal(got_ids[0::2], base_ids[0::2])
    assert bool((got_ids[1::2] <= 10).all())                      # EOS or a digit (ids 1..10)


def test_graph_host_crops_and_super_chunks():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 25, 13, decode_ar=True, refine_iters=1)
    rng = np.random.default_rng(5)
    allow = [[DIGITS, "abc", None, "", DIGITS + "xyz"][b % 5] for b in range(1024)]
    x = synth_images(cfg, 1024, 142).cuda()
    mask = m.allowlist_mask(allow, 1024)
    full, full_ids = _run(m, x, mask)
    lo, lo_ids = _run(m, x[:512], mask[:512])
    hi, hi_ids = _run(m, x[512:], mask[512:])
    assert _same(full, torch.cat([lo, hi])) and torch.equal(full_ids, torch.cat([lo_ids, hi_ids]))
    m.model.set_engine_option("use_graph", 0)
    eager, eager_ids = _run(m, x[:512], mask[:512])
    m.model.set_engine_option("use_graph", 1)
    assert _same(eager, lo) and torch.equal(eager_ids, lo_ids)
    # raw crops: device entry point == host entry point == the preprocessed uint8 stack, graph and eager
    crops = [torch.from_numpy(rng.integers(0, 256, (int(rng.integers(16, 129)), int(rng.integers(32, 513)), 3),
                                           dtype=np.uint8)) for _ in range(300)]
    cmask = m.allowlist_mask(allow[:300], 300)
    with torch.inference_mode():
        stack = m.preprocess(crops)
    dev, dev_ids = _run(m, [c.cuda() for c in crops], cmask)
    host, host_ids = _run(m, crops, cmask)
    u8, u8_ids = _run(m, stack, cmask)
    assert _same(dev, u8) and torch.equal(dev_ids, u8_ids)
    assert _same(host, u8.cpu()) and torch.equal(host_ids, u8_ids.cpu())
    with torch.inference_mode():
        assert _same(m(crops, allowlist=allow[:300]), host)
        assert _same(m([c.cuda() for c in crops], allowlist=allow[:300]), dev)
        assert _same(m(stack, allowlist=allow[:300]), u8)


@pytest.mark.parametrize("arch", ["parseq", "vitstr"])
def test_nan_crop_with_digits_mask_decodes_to_eos(arch):
    from parseq_b200.weights import synth_images
    kw = {} if arch == "vitstr" else {"decode_ar": True, "refine_iters": 1}
    cfg, sd, m = _model(arch, 25, 14, **kw)
    x = synth_images(cfg, 6, 143).cuda()
    allow = [DIGITS, None, "abc", DIGITS, None, "xyz"]
    mask = m.allowlist_mask(allow, 6)
    base, base_ids = _run(m, x, mask)
    x[3] = float("nan")
    got, got_ids = _run(m, x, mask)
    keep = [0, 1, 2, 4, 5]
    assert _same(got[keep], base[keep]) and torch.equal(got_ids[keep], base_ids[keep])
    assert int(got_ids[3, 0]) == 0
    labels, _ = m.postprocess(got)
    assert labels[3] == ""
