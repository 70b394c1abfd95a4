"""GPU: models with long labels (max_label_length 32..63, L = 33..64 decode positions).  The decoder's id rows are 64 wide:
the cluster AR kernel runs its 64-pitch instantiations (dec_ar2.cuh, IDP = 64), the chain of separate kernels runs the
two-keys-per-lane self-attention, and heads of 97..128 classes run the AR loop as a chain.  Checked against the
reference goldens (tests/golden/long), against the chain (ar_kernel = 0), and for the properties that need no reference:
ids are the first maxima of the logits, rows do not depend on the batch, graph replay equals eager."""
import glob
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "long")
TOL_FP32_MAX = 2.0e-2          # the bounds of test_gpu_parity.py
TOL_FP32_MEAN = 3.0e-3
TAU = 2.0e-2
PARSEQ_CASES = sorted(p for p in glob.glob(os.path.join(GOLDEN, "long_*.pt"))
                      if not os.path.basename(p).startswith("long_vitstr"))


def _model(experiment, mll, seed, n_extra=0, img_size=(32, 128), sd_edit=None, sharp=0.0, **kw):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config_long(experiment, mll, n_extra, img_size)
    sd = init_state_dict(cfg, seed, sharp=sharp)
    if sd_edit is not None:
        sd_edit(sd)
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=mll, img_size=list(img_size), **kw)
    (m if experiment == "vitstr" else m.model).load_state_dict(sd)
    return cfg, sd, m.eval().to("cuda")


def _forced_from_blob(blob, L):
    forced = forced_refine = None
    if blob["ar_ids"] is not None:
        forced = torch.zeros((blob["batch"], L), dtype=torch.int32)
        forced[:, : blob["ar_ids"].shape[1]] = blob["ar_ids"]
    if blob["refine_ctx"]:
        forced_refine = torch.zeros((len(blob["refine_ctx"]), blob["batch"], L), dtype=torch.int32)
        for r, c in enumerate(blob["refine_ctx"]):
            forced_refine[r, :, : c.shape[1]] = c
    return forced, forced_refine


def _bos_forced(ids, bos):
    """AR teacher forcing that replays a run's own tokens: position 0 is BOS, position i + 1 the id emitted at step i."""
    f = torch.empty_like(ids)
    f[:, 0] = bos
    f[:, 1:] = ids[:, :-1]
    return f


def _close(a, b):
    err = (a - b).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN, (err.max().item(), err.mean().item())


def test_label_length_limits():
    from parseq_b200.engine import EngineError
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny", 63, 1, decode_ar=True, refine_iters=0)
    x = synth_images(cfg, 2, 90).cuda()
    with torch.inference_mode():
        logits, ids = m.model.forward(m.tokenizer, x, 63, return_ids=True)
    assert logits.shape == (2, 64, 95) and torch.equal(ids.long(), logits.argmax(-1))
    with pytest.raises(EngineError, match="max_label_length <= 31"):
        m.model.set_engine_option("ar_kernel", 1)
    from parseq_b200.factory import create_model
    big = create_model("parseq-tiny", max_label_length=64).eval().to("cuda")
    with pytest.raises(EngineError, match="63"):
        big.model.engine()


@pytest.mark.parametrize("mode", ["default", "fused_ln", "ar_chain"])
@pytest.mark.parametrize("path", PARSEQ_CASES, ids=lambda p: os.path.basename(p)[:-3])
def test_teacher_forced_vs_reference_golden(path, mode):
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(path, weights_only=False)
    cfg, sd, m = _model(blob["experiment"], blob["max_label_length"], blob["weight_seed"], blob["n_extra"],
                        tuple(blob["img_size"]), decode_ar=blob["decode_ar"], refine_iters=blob["refine_iters"])
    assert state_dict_digest(sd) == blob["sd_digest"]
    if mode == "fused_ln":
        m.model.set_engine_option("fuse_ln", 7)
    elif mode == "ar_chain":
        m.model.set_engine_option("ar_kernel", 0)
    x = synth_images(cfg, blob["batch"], blob["image_seed"])
    L = m.model.engine().num_steps(blob["max_length"])
    forced, forced_refine = _forced_from_blob(blob, L)
    with torch.inference_mode():
        logits = m.model.forward(m.tokenizer, x.cuda(), blob["max_length"], forced_ids=forced,
                                 forced_refine=forced_refine).cpu()
    ref = blob["logits"]
    assert logits.shape == ref.shape
    _close(logits, ref)
    top2 = ref.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > TAU
    assert bool((logits.argmax(-1) == ref.argmax(-1))[clear].all())


def test_vitstr_vs_reference_golden():
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(os.path.join(GOLDEN, "long_vitstr_s_b1.pt"), weights_only=False)
    cfg, sd, m = _model("vitstr", blob["max_label_length"], blob["weight_seed"], blob["n_extra"])
    assert state_dict_digest(sd) == blob["sd_digest"]
    x = synth_images(cfg, blob["batch"], blob["image_seed"])
    with torch.inference_mode():
        logits, ids = m.model.forward_tokens(x.cuda(), blob["max_length"], return_ids=True)
    logits, ids = logits.cpu(), ids.cpu()
    assert logits.shape == blob["logits"].shape == (1, 64, 95)
    _close(logits, blob["logits"])
    assert torch.equal(ids.long(), logits.argmax(-1))


REFINE_CASES = sorted(glob.glob(os.path.join(GOLDEN, "eos_*.pt")))


@pytest.mark.parametrize("mode", ["default", "fused_ln"])
@pytest.mark.parametrize("path", REFINE_CASES, ids=lambda p: os.path.basename(p)[:-3])
def test_refine_with_eos_in_either_key_group_vs_reference_golden(path, mode):
    """The cloze pass at L = 64 on a given context whose first EOS is at 3..63 or absent (sharp-attention weights): the
    padding mask from the first EOS, found from one ballot per 32 keys, against the reference."""
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(path, weights_only=False)
    cfg, sd, m = _model(blob["experiment"], 63, blob["weight_seed"], 0, tuple(blob["img_size"]), sharp=blob["sharp"],
                        decode_ar=False, refine_iters=1)
    assert state_dict_digest(sd) == blob["sd_digest"]
    if mode == "fused_ln":
        m.model.set_engine_option("fuse_ln", 7)
    x = synth_images(cfg, blob["batch"], blob["image_seed"])
    with torch.inference_mode():
        logits = m.model.forward(m.tokenizer, x.cuda(), 63, forced_refine=blob["refine_ctx"][0][None]).cpu()
    ref = blob["logits"]
    assert logits.shape == ref.shape == (5, 64, 95)
    for b in range(ref.shape[0]):
        _close(logits[b], ref[b])
    top2 = ref.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > TAU
    assert bool((logits.argmax(-1) == ref.argmax(-1))[clear].all())


# (experiment, extra characters, batch, engine options, expected (cluster size, MT, head split, wide); None = any)
AR_PATHS = {
    "d384_cs8_mt1":  ("parseq",             0,    40, {"ar_cluster_size": 8}, (8, 1, 0, 0)),
    "d384_cs6_mt1":  ("parseq",             0,    40, {"ar_cluster_size": 6}, (6, 1, 0, 0)),
    "d384_cs8_mt2":  ("parseq",             0,    60, {"ar_cluster_size": 8, "ar_clusters": 2}, (8, 2, 0, 0)),
    "d384_cs6_mt2":  ("parseq",             0,    60, {"ar_cluster_size": 6, "ar_clusters": 2}, (6, 2, 0, 0)),
    "d384_hs":       ("parseq",             0,    1,  {}, (8, 1, 1, 0)),
    "d192_cs8_mt2":  ("parseq-tiny",        0,    60, {"ar_cluster_size": 8, "ar_clusters": 2}, (8, 2, 0, 0)),
    "d192_hs":       ("parseq-tiny",        0,    3,  {}, (8, 1, 1, 0)),
    "d192_wide":     ("parseq-tiny",        2906, 60, {}, (None, None, 0, 1)),
    "d384_wide_hs":  ("parseq",             2906, 1,  {}, (8, 1, 1, 1)),
    "d768_cs8":      ("parseq-base-48x160", 0,    20, {"ar_cluster_size": 8}, (8, 1, 0, 0)),
    "d768_cs6":      ("parseq-base-48x160", 0,    20, {"ar_cluster_size": 6}, (6, 1, 0, 0)),
}


@pytest.mark.parametrize("path", list(AR_PATHS))
def test_ar_paths_agree_with_the_chain(path):
    from parseq_b200.weights import synth_images
    exp, n_extra, B, opts, want = AR_PATHS[path]
    img = (48, 160) if exp == "parseq-base-48x160" else (32, 128)
    cfg, sd, m = _model(exp, 63, 7, n_extra, img, decode_ar=True, refine_iters=0)
    x = synth_images(cfg, B, 91).cuda()
    eng = m.model.engine()
    with torch.inference_mode():
        m.model.set_engine_option("ar_kernel", 0)
        chain, chain_ids = m.model.forward(m.tokenizer, x, 63, return_ids=True)
        forced = _bos_forced(chain_ids, m.bos_id)
        assert torch.equal(m.model.forward(m.tokenizer, x, 63, forced_ids=forced), chain)
        m.model.set_engine_option("ar_kernel", 2)
        for k, v in opts.items():
            m.model.set_engine_option(k, v)
        cluster = m.model.forward(m.tokenizer, x, 63, forced_ids=forced)
    got = tuple(eng.debug_int(k) for k in ("ar_last_cluster_size", "ar_last_mt", "ar_last_head_split", "ar_last_wide"))
    assert all(w is None or w == g for w, g in zip(want, got)), (want, got)
    assert eng.debug_int("ar_last_ids_pitch") == 64
    assert cluster.shape == (B, 64, cfg.num_classes)
    _close(cluster.cpu(), chain.cpu())


@pytest.mark.parametrize("experiment,n_extra,B", [("parseq", 0, 1), ("parseq", 0, 37), ("parseq-tiny", 2906, 5),
                                                  ("parseq", 15, 9)])
def test_free_running_ids_are_first_maxima_and_replay_bit_identically(experiment, n_extra, B):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(experiment, 63, 3, n_extra, decode_ar=True, refine_iters=0)
    x = synth_images(cfg, B, 92).cuda()
    with torch.inference_mode():
        logits, ids = m.model.forward(m.tokenizer, x, 63, return_ids=True)
        assert torch.equal(ids.long(), logits.argmax(-1))
        again = m.model.forward(m.tokenizer, x, 63, forced_ids=_bos_forced(ids, m.bos_id))
    assert torch.equal(again, logits)


@pytest.mark.parametrize("route", ["cs6", "cs8", "chain"])
def test_rows_do_not_depend_on_the_batch(route):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 63, 5, decode_ar=True, refine_iters=1)
    if route == "chain":
        m.model.set_engine_option("ar_kernel", 0)
    else:
        m.model.set_engine_option("ar_cluster_size", int(route[2:]))
    x = synth_images(cfg, 48, 93).cuda()
    with torch.inference_mode():
        full, full_ids = m.model.forward(m.tokenizer, x, 63, return_ids=True)
        for lo, hi in ((0, 1), (5, 8), (17, 40)):
            part, part_ids = m.model.forward(m.tokenizer, x[lo:hi], 63, return_ids=True)
            assert torch.equal(part, full[lo:hi]) and torch.equal(part_ids, full_ids[lo:hi])


@pytest.mark.parametrize("B", [3, 512])
def test_graph_replay_equals_eager(B):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 63, 6, decode_ar=True, refine_iters=1)
    x = synth_images(cfg, B, 94).cuda()
    with torch.inference_mode():
        m.model.set_engine_option("use_graph", 1)
        g1 = m.model.forward(m.tokenizer, x, 63)
        g2 = m.model.forward(m.tokenizer, x, 63)
        m.model.set_engine_option("use_graph", 0)
        eager = m.model.forward(m.tokenizer, x, 63)
    assert torch.equal(g1, eager) and torch.equal(g2, eager)


def test_max_length_below_the_limit_and_early_exit():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 63, 8, decode_ar=True, refine_iters=0)
    x = synth_images(cfg, 4, 95).cuda()
    with torch.inference_mode():
        full, ids = m.model.forward(m.tokenizer, x, 63, return_ids=True)
        short = m.model.forward(m.tokenizer, x, 40)
        assert short.shape == (4, 41, 95)
        assert torch.equal(short, full[:, :41])          # the first 41 AR steps do not depend on L
        # early exit (max_length=None, no refinement): S = the last first-EOS over the batch, found on the device
        forced = _bos_forced(ids, m.bos_id)
        forced[:, 1:] = torch.where(forced[:, 1:] == 0, torch.ones_like(forced[:, 1:]), forced[:, 1:])
        forced[0, 21] = 0                                 # step 20 emits EOS in image 0
        forced[1, 38] = 0                                 # step 37 emits EOS in image 1
        forced[2, 45] = 0
        forced[3, 50] = 0
        exited = m.model.forward(m.tokenizer, x, None, forced_ids=forced)
        longest = m.model.forward(m.tokenizer, x, 63, forced_ids=forced)
    assert exited.shape == (4, 50, 95)
    assert torch.equal(exited, longest[:, :50])


def test_decode_api_with_64_queries_and_masks():
    from oracle.parseq_oracle import ParseqOracle
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 63, 12)
    o = ParseqOracle(cfg, sd, "fp32")
    B, L = 3, 64
    g = torch.Generator().manual_seed(5)
    x = synth_images(cfg, B, 96)
    memory = o.encode(x)
    tgt = torch.randint(1, 95, (B, L), generator=g)
    tgt[:, 0] = cfg.num_tokens - 2
    qmask = torch.zeros((L, L), dtype=torch.bool)
    qmask[torch.arange(L - 1), torch.arange(1, L)] = True                       # model.py:157
    qmask[:, 40] = True                                                         # a masked key past 32
    pmask = torch.rand((B, L), generator=g) < 0.3
    pmask[:, 0] = False
    ref = o._decode(tgt, memory, o.p["pos_queries"][:, :L].expand(B, -1, -1), qmask, pmask)
    with torch.inference_mode():
        out = m.model.decode(tgt.cuda(), memory.cuda(), tgt_query_mask=qmask.cuda(), tgt_padding_mask=pmask.cuda())
        logits = m.model.head(out).cpu()
    assert out.shape == (B, L, cfg.embed_dim)
    _close(logits, ref)


def test_postprocess_matches_tokenizer_decode():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 63, 9, sd_edit=lambda sd: sd["head.bias"].add_(
        torch.linspace(0, 2, sd["head.bias"].numel())), decode_ar=True, refine_iters=1)
    x = synth_images(cfg, 6, 97).cuda()
    with torch.inference_mode():
        logits = m.model.forward(m.tokenizer, x, 63)
        labels, confs = m.postprocess(logits)
        ref_labels, ref_probs = m.tokenizer.decode(logits.softmax(-1))
    assert logits.shape[1] == 64
    assert labels == ref_labels
    for c, p in zip(confs, ref_probs):
        assert abs(float(c) - float(p.prod())) <= 1e-4 * max(1.0, float(p.prod()))


@pytest.mark.parametrize("route", ["cluster", "chain"])
def test_nan_crop_leaves_the_other_images_bit_identical(route):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 63, 10, decode_ar=True, refine_iters=1)
    if route == "chain":
        m.model.set_engine_option("ar_kernel", 0)
    x = synth_images(cfg, 5, 98).cuda()
    with torch.inference_mode():
        clean, clean_ids = m.model.forward(m.tokenizer, x, 63, return_ids=True)
        x[2, :, 5:9, 10:20] = float("nan")
        dirty, dirty_ids = m.model.forward(m.tokenizer, x, 63, return_ids=True)
    keep = [0, 1, 3, 4]
    assert torch.equal(dirty[keep], clean[keep]) and torch.equal(dirty_ids[keep], clean_ids[keep])
