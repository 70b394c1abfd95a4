"""Generates tests/golden/depth/*.pt: golden outputs of the reference's own modules (strhub.models.parseq.model.PARSeq
under oracle/timm_shim.py) for PARSeq decoders of depth 2 and 3.  Run where the reference tree exists:

    python tests/make_golden_depth.py

Weights are not stored: they are regenerated from (experiment, seed, geometry) by parseq_b200.weights.init_state_dict
and verified through `sd_digest`.  The goldens live in a subdirectory of their own, away from the globs of the
depth-1 parity tests.  Every golden is checked against the fp64 depth-N oracle (tests/dec_depth_oracle.py).
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from make_golden_long import charset, cloze_masks, make_config_long, refine_context   # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images, state_dict_digest     # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "depth")
GOLDEN_FILE_LIMIT = 1_000_000
FP64_TOL = 1e-5
REFINE_FP64_TOL = 5e-5       # sharp weights: the longest sums (as tests/make_golden_long.py)

# (case name, experiment, dec_depth, max_label_length, extra characters, weight seed, batch, image seed, decode_ar,
#  refine_iters, max_length)
CASES = [
    ("d2_ti_ar1_b2",       "parseq-tiny", 2, 25, 0,    90, 2, 100, True,  1, None),
    ("d2_s_nar2_b2",       "parseq",      2, 25, 0,    91, 2, 101, False, 2, None),
    ("d3_s_ar0_b2",        "parseq",      3, 25, 0,    92, 2, 102, True,  0, None),   # batch-wide early exit S
    ("d2_s_l64_ar1_b1",    "parseq",      2, 63, 0,    93, 1, 103, True,  1, None),   # id pitch 64, two keys per lane
    ("d2_ti_c3001_ar1_b1", "parseq-tiny", 2, 25, 2906, 94, 1, 104, True,  1, None),   # head tail of > 128 classes
    ("d2_s_len5_ar1_b2",   "parseq",      2, 25, 0,    95, 2, 105, True,  1, 5),      # max_length < max_label_length
]
# cloze refinement on a chosen context whose first EOS lies in either 32-key group (L = 64), sharp weights:
# (case name, experiment, dec_depth, weight seed, sharpness, image seed, EOS positions per image)
REFINE_CASES = [
    ("d2_eos_s_refine_b4", "parseq", 2, 96, 4.0, 106, [[7], [32], [40, 55], []]),
]
# PARSeq.decode with caller masks: (case name, experiment, dec_depth, weight seed, batch, image seed, J, NQ, mask seed)
DECODE_CASES = [
    ("d2_decode_ti_b3", "parseq-tiny", 2, 97, 3, 107, 9, 7, 5),
]


def _save(blob, name):
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    return size


def _common(name, exp, depth, mll, n_extra, img, wseed, B, iseed, sd):
    return dict(name=name, experiment=exp, dec_depth=depth, max_label_length=mll, img_size=list(img), n_extra=n_extra,
                weight_seed=wseed, batch=B, image_seed=iseed, sd_digest=state_dict_digest(sd))


def make_parseq():
    from oracle import reference_loader as RL
    from dec_depth_oracle import DepthOracle
    for name, exp, depth, mll, n_extra, wseed, B, iseed, ar, ri, ml in CASES:
        cfg = make_config_long(exp, mll, n_extra, dec_depth=depth)
        sd = init_state_dict(cfg, wseed)
        ref, tok = RL.build_reference_model(cfg, sd)
        x = synth_images(cfg, B, iseed)
        ref.decode_ar, ref.refine_iters = ar, ri
        with torch.inference_mode():
            logits = ref(tok, x, ml).clone()
        o = DepthOracle(cfg, sd, "fp64").forward(x, ml, ar, ri)
        assert o.logits.shape == logits.shape, (name, o.logits.shape, logits.shape)
        err = (o.logits.float() - logits).abs().max().item()
        assert err < FP64_TOL, (name, err)
        blob = _common(name, exp, depth, mll, n_extra, cfg.img_size, wseed, B, iseed, sd)
        blob.update(decode_ar=ar, refine_iters=ri, max_length=ml, logits=logits.contiguous(),
                    min_margin_fp64=o.min_margin.float(), steps=o.steps,
                    ar_ids=None if o.ar_ids is None else o.ar_ids.int(), refine_ctx=[c.int() for c in o.refine_ctx],
                    source="reference strhub.models.parseq.model.PARSeq (timm shim), torch %s CPU fp32" % torch.__version__)
        size = _save(blob, name)
        print(f"{name:22s} depth={depth} L={mll + 1} C={cfg.num_classes} logits {tuple(logits.shape)} S={o.steps} "
              f"|ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


def make_refine():
    from oracle import reference_loader as RL
    from dec_depth_oracle import DepthOracle
    for name, exp, depth, wseed, sharp, iseed, eos in REFINE_CASES:
        cfg = make_config_long(exp, 63, 0, dec_depth=depth)
        sd = init_state_dict(cfg, wseed, sharp=sharp)
        ref, tok = RL.build_reference_model(cfg, sd)
        B, L = len(eos), 64
        x = synth_images(cfg, B, iseed)
        ref.decode_ar, ref.refine_iters = False, 0
        with torch.inference_mode():
            nar = ref(tok, x, 63)
            ctx = refine_context(nar.argmax(-1), tok.bos_id, eos)
            qmask, pmask = cloze_masks(ctx)
            memory = ref.encode(x)
            pos_queries = ref.pos_queries[:, :L].expand(B, -1, -1)
            # model.py:157-165: the content stream runs under the same cloze mask as the query stream
            logits = ref.head(ref.decode(ctx, memory, qmask, pmask, pos_queries, qmask)).clone()
        o = DepthOracle(cfg, sd, "fp64")
        olog = o._decode(ctx, o.encode(x), o.p["pos_queries"][:, :L].expand(B, -1, -1), qmask, pmask, qmask).float()
        err = (olog - logits).abs().max().item()
        assert err < REFINE_FP64_TOL, (name, err)
        blob = _common(name, exp, depth, 63, 0, cfg.img_size, wseed, B, iseed, sd)
        blob.update(sharp=sharp, decode_ar=False, refine_iters=1, max_length=63, eos_positions=eos,
                    refine_ctx=[ctx.int()], logits=logits.contiguous(),
                    source="reference strhub.models.parseq.model.PARSeq (timm shim) refinement step on a given context, "
                           "torch %s CPU fp32" % torch.__version__)
        size = _save(blob, name)
        print(f"{name:22s} depth={depth} L={L} logits {tuple(logits.shape)} |ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


def decode_inputs(cfg, B, J, NQ, mseed, bos):
    """Context ids, custom queries, a random content mask, a random query mask and a padding mask.  Content row J - 2
    sees key J - 1 only, which image 2 pads: there every key of that row is masked, the reference's softmax yields NaN,
    and the NaN K/V row it feeds to the next layer turns every output of image 2 into NaN (0 * NaN in P.V)."""
    g = torch.Generator().manual_seed(mseed)
    ids = torch.randint(0, cfg.num_classes + 1, (B, J), generator=g)
    ids[:, 0] = bos
    query = torch.randn((B, NQ, cfg.embed_dim), generator=g)
    cmask = torch.rand((J, J), generator=g) < 0.3
    cmask[:, 0] = False
    cmask[J - 2, :] = True
    cmask[J - 2, J - 1] = False
    qmask = torch.rand((NQ, J), generator=g) < 0.3
    qmask[:, 0] = False
    pmask = torch.zeros((B, J), dtype=torch.bool)
    pmask[1, 3] = True
    pmask[2, J - 1] = True
    return ids, query, cmask, qmask, pmask


def make_decode():
    from oracle import reference_loader as RL
    from dec_depth_oracle import DepthOracle
    for name, exp, depth, wseed, B, iseed, J, NQ, mseed in DECODE_CASES:
        cfg = make_config_long(exp, 25, 0, dec_depth=depth)
        sd = init_state_dict(cfg, wseed)
        ref, tok = RL.build_reference_model(cfg, sd)
        x = synth_images(cfg, B, iseed)
        ids, query, cmask, qmask, pmask = decode_inputs(cfg, B, J, NQ, mseed, tok.bos_id)
        with torch.inference_mode():
            memory = ref.encode(x)
            out = ref.decode(ids, memory, cmask, pmask, query, qmask).clone()
            out_nomask = ref.decode(ids, memory, None, pmask, query, qmask).clone()
        o = DepthOracle(cfg, sd, "fp64")
        mem = o.encode(x)
        oo = o.decoder_out(ids, mem, query.double(), qmask, pmask, cmask).float()
        assert torch.equal(torch.isnan(oo), torch.isnan(out)), name
        fin = ~torch.isnan(out)
        err = (oo[fin] - out[fin]).abs().max().item()
        assert err < FP64_TOL, (name, err)
        blob = _common(name, exp, depth, 25, 0, cfg.img_size, wseed, B, iseed, sd)
        blob.update(ids=ids.int(), query=query, content_mask=cmask, query_mask=qmask, padding_mask=pmask,
                    memory=memory.clone(), out=out, out_no_content_mask=out_nomask,
                    source="reference PARSeq.decode (timm shim), torch %s CPU fp32" % torch.__version__)
        size = _save(blob, name)
        print(f"{name:22s} depth={depth} out {tuple(out.shape)} NaN rows {int(torch.isnan(out).any(-1).sum())} "
              f"|ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


def make_keys():
    from oracle import reference_loader as RL
    cfg = make_config_long("parseq", 25, 0, dec_depth=2)
    ref, _ = RL.build_reference_model(cfg, init_state_dict(cfg, 0))
    keys = {k: list(v.shape) for k, v in ref.state_dict().items()}
    torch.save(dict(experiment="parseq", dec_depth=2, keys=keys), os.path.join(OUT, "d2_s_state_dict_keys.pt"))
    print(f"state_dict keys at depth 2: {len(keys)}")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    make_keys()
    make_decode()
    make_parseq()
    make_refine()
