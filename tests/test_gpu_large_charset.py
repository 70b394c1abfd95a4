"""GPU: models with a large character set (> 128 head classes).  The AR loop runs on the cluster kernel's class-sliced head
(dec_ar2.cuh, WIDE): each CTA of a cluster owns a slice of the classes and the greedy token is merged across the cluster.
Checked against the reference goldens (tests/golden/cjk), against the chain of separate kernels (ar_kernel = 0), and for
the properties that need no reference: ids equal the first maximum of the logits, exact ties go to the lower class index
wherever the tied pair lies, rows do not depend on the batch, graph replay equals eager."""
import glob
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cjk")
TOL_FP32_MAX = 2.0e-2          # the bounds of test_gpu_parity.py
TOL_FP32_MEAN = 3.0e-3
TAU = 2.0e-2
PARSEQ_CASES = sorted(p for p in glob.glob(os.path.join(GOLDEN, "cjk_*.pt"))
                      if not os.path.basename(p).startswith(("cjk_vitstr", "cjk_tokenizer")))


def _model(experiment, n_cjk, seed, sd_edit=None, **kw):
    from make_golden_cjk import cjk_charset, make_config_cjk
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config_cjk(experiment, n_cjk)
    sd = init_state_dict(cfg, seed)
    if sd_edit is not None:
        sd_edit(sd)
    m = create_model(experiment, charset_train=cjk_charset(n_cjk), **kw)
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


@pytest.mark.parametrize("mode", ["default", "fused_ln", "ar_chain"])
@pytest.mark.parametrize("path", PARSEQ_CASES, ids=lambda p: os.path.basename(p)[:-3])
def test_teacher_forced_vs_reference_golden(path, mode):
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(path, weights_only=False)
    cfg, sd, m = _model(blob["experiment"], blob["n_cjk"], blob["weight_seed"], decode_ar=blob["decode_ar"],
                        refine_iters=blob["refine_iters"])
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
    err = (logits - ref).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN, (err.max().item(), err.mean().item())
    top2 = ref.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > TAU
    assert bool((logits.argmax(-1) == ref.argmax(-1))[clear].all())


def test_vitstr_vs_reference_golden():
    from parseq_b200.weights import synth_images, state_dict_digest
    blob = torch.load(os.path.join(GOLDEN, "cjk_vitstr_s_b1.pt"), weights_only=False)
    cfg, sd, m = _model("vitstr", blob["n_cjk"], blob["weight_seed"])
    assert state_dict_digest(sd) == blob["sd_digest"]
    x = synth_images(cfg, blob["batch"], blob["image_seed"])
    with torch.inference_mode():
        logits, ids = m.model.forward_tokens(x.cuda(), blob["max_length"], return_ids=True)
    logits, ids = logits.cpu(), ids.cpu()
    ref = blob["logits"]
    err = (logits - ref).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN
    assert torch.equal(ids.long(), logits.argmax(-1))


def _bos_forced(ids, bos):
    """AR teacher forcing that replays a run's own tokens: position 0 is BOS, position i + 1 the id emitted at step i."""
    f = torch.empty_like(ids)
    f[:, 0] = bos
    f[:, 1:] = ids[:, :-1]
    return f


@pytest.mark.parametrize("experiment,n_cjk,B", [("parseq", 2906, 1), ("parseq", 2906, 37), ("parseq-tiny", 6905, 5)])
def test_free_running_ids_are_first_maxima_and_replay_bit_identically(experiment, n_cjk, B):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model(experiment, n_cjk, 3, decode_ar=True, refine_iters=0)
    x = synth_images(cfg, B, 60).cuda()
    with torch.inference_mode():
        logits, ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
        assert torch.equal(ids.long(), logits.argmax(-1))
        again = m.model.forward(m.tokenizer, x, 25, forced_ids=_bos_forced(ids, m.bos_id))
    assert torch.equal(again, logits)


def _tie(i, j):
    def edit(sd):
        w, b = sd["head.weight"].clone(), sd["head.bias"].clone()
        w[j] = w[i]
        b[i] = b[j] = 50.0
        sd["head.weight"], sd["head.bias"] = w, b
    return edit


# PARSeq-S with C = 3001: clusters of 8 own 376 classes each (6: 504), in chunks of 128
TIES = {"cta_slices": (10, 400), "chunks_of_one_slice": (380, 510), "one_chunk": (3, 100)}


@pytest.mark.parametrize("B", [1, 64])
@pytest.mark.parametrize("where", list(TIES))
def test_exact_ties_go_to_the_lower_index(where, B):
    from parseq_b200.weights import synth_images
    i, j = TIES[where]
    cfg, sd, m = _model("parseq", 2906, 4, sd_edit=_tie(i, j), decode_ar=True, refine_iters=1)
    x = synth_images(cfg, B, 61).cuda()
    with torch.inference_mode():
        logits, ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
        assert bool((ids == i).all())
        # the AR loop itself picked i at every step: replaying i as the context reproduces its logits
        m.model.refine_iters = 0
        ar_logits, ar_ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
        assert bool((ar_ids == i).all())
        forced = torch.full_like(ar_ids, i)
        forced[:, 0] = m.bos_id
        assert torch.equal(m.model.forward(m.tokenizer, x, 25, forced_ids=forced), ar_logits)
        m.model.decode_ar = False
        nar_logits, nar_ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
        assert bool((nar_ids == i).all())
        assert bool((logits[..., i] == logits[..., j]).all())


@pytest.mark.parametrize("cs", [6, 8])
def test_rows_do_not_depend_on_the_batch(cs):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 2906, 5, decode_ar=True, refine_iters=1)
    m.model.set_engine_option("ar_cluster_size", cs)
    x = synth_images(cfg, 48, 62).cuda()
    with torch.inference_mode():
        full, full_ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
        for lo, hi in ((0, 1), (5, 8), (17, 40)):
            part, part_ids = m.model.forward(m.tokenizer, x[lo:hi], 25, return_ids=True)
            assert torch.equal(part, full[lo:hi]) and torch.equal(part_ids, full_ids[lo:hi])


@pytest.mark.parametrize("B", [3, 512])
def test_graph_replay_equals_eager(B):
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 2906, 6, decode_ar=True, refine_iters=1)
    x = synth_images(cfg, B, 63).cuda()
    with torch.inference_mode():
        m.model.set_engine_option("use_graph", 1)
        g1 = m.model.forward(m.tokenizer, x, 25)
        g2 = m.model.forward(m.tokenizer, x, 25)
        m.model.set_engine_option("use_graph", 0)
        eager = m.model.forward(m.tokenizer, x, 25)
    assert torch.equal(g1, eager) and torch.equal(g2, eager)


def test_cluster_kernel_agrees_with_the_chain():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 2906, 7, decode_ar=True, refine_iters=0)
    x = synth_images(cfg, 40, 64).cuda()
    with torch.inference_mode():
        m.model.set_engine_option("ar_kernel", 0)
        chain, chain_ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
        forced = _bos_forced(chain_ids, m.bos_id)
        chain_f = m.model.forward(m.tokenizer, x, 25, forced_ids=forced)
        m.model.set_engine_option("ar_kernel", 2)
        cluster = m.model.forward(m.tokenizer, x, 25, forced_ids=forced)
    assert torch.equal(chain_f, chain)
    err = (cluster - chain).abs()
    assert err.max().item() <= TOL_FP32_MAX and err.mean().item() <= TOL_FP32_MEAN


def test_class_limits():
    from parseq_b200.engine import EngineError
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq-tiny", 16289, 8, decode_ar=True, refine_iters=0)      # 16384 classes
    assert cfg.num_classes == 16384
    x = synth_images(cfg, 2, 65).cuda()
    with torch.inference_mode():
        logits, ids = m.model.forward(m.tokenizer, x, 25, return_ids=True)
    assert logits.shape == (2, 26, 16384) and torch.equal(ids.long(), logits.argmax(-1))
    with pytest.raises(EngineError, match="ar_kernel = 1"):
        m.model.set_engine_option("ar_kernel", 1)
    from make_golden_cjk import cjk_charset
    from parseq_b200.factory import create_model
    big = create_model("parseq-tiny", charset_train=cjk_charset(16290)).eval().to("cuda")
    with pytest.raises(EngineError, match="16384"):
        big.model.engine()


def test_postprocess_matches_tokenizer_decode():
    from parseq_b200.weights import synth_images
    cfg, sd, m = _model("parseq", 2906, 9, sd_edit=lambda sd: sd["head.bias"].add_(
        torch.linspace(0, 2, sd["head.bias"].numel())), decode_ar=True, refine_iters=1)
    x = synth_images(cfg, 6, 66).cuda()
    with torch.inference_mode():
        logits = m.model.forward(m.tokenizer, x, 25)
        labels, confs = m.postprocess(logits)
        ref_labels, ref_probs = m.tokenizer.decode(logits.softmax(-1))
    assert labels == ref_labels
    for c, p in zip(confs, ref_probs):
        assert abs(float(c) - float(p.prod())) <= 1e-4 * max(1.0, float(p.prod()))
