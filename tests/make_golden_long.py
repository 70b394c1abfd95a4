"""Generates tests/golden/long/*.pt: golden outputs of the reference's own modules (strhub.models.parseq.model.PARSeq and
strhub.models.vitstr.model.ViTSTR under oracle/timm_shim.py) for models with long labels (max_label_length 40..63, i.e.
33..64 decode positions).  Run where the reference tree exists:

    python tests/make_golden_long.py

Weights are not stored: they are regenerated from (experiment, seed, geometry) by parseq_b200.weights.init_state_dict
and verified through `sd_digest`.  The goldens live in a subdirectory of their own: the PARSeq and ViTSTR parity tests
glob the files at the top of tests/golden and build 25-character models for them.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from parseq_b200.config import CHARSET_94, make_config               # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images, state_dict_digest  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "long")
GOLDEN_FILE_LIMIT = 1_000_000


def charset(n_extra: int) -> str:
    """The 94 characters of 94_full followed by n_extra CJK ideographs (head classes: 95 + n_extra)."""
    return CHARSET_94 + "".join(chr(0x4E00 + i) for i in range(n_extra))


# (case name, experiment, max_label_length, image (H, W), extra characters, weight seed, batch, image seed, decode_ar,
#  refine_iters, max_length)
CASES = [
    ("long_s_w256_ar1_b2",   "parseq",      63, (32, 256), 0,    70, 2, 80, True,  1, None),   # T = 256, the long-line crop
    ("long_ti_nar2_b1",      "parseq-tiny", 47, (32, 128), 0,    71, 1, 81, False, 2, None),
    ("long_s_ar0_b2",        "parseq",      40, (32, 128), 0,    72, 2, 82, True,  0, None),   # batch-wide early exit S
    ("long_ti_c3001_ar1_b1", "parseq-tiny", 63, (32, 128), 2906, 73, 1, 83, True,  1, None),   # class-sliced head
    ("long_s_c110_ar1_b2",   "parseq",      48, (32, 128), 15,   74, 2, 84, True,  1, None),   # 97..128 classes: chain
]
# (case name, max_label_length, extra characters, weight seed, batch, image seed, max_length)
VITSTR_CASES = [
    ("long_vitstr_s_b1", 63, 0, 75, 1, 85, None),
]


# Cloze refinement with a caller-chosen context (forced_refine) whose first EOS lies in either 32-key group of the
# self-attention, on sharp-attention weights, so that the padding mask from the first EOS is checked against the
# reference at L = 64 (D = 768 at a lower sharpness: at 4.0 its bf16 rounding alone moves the logits past the engine's
# tolerance): (case name, experiment, image (H, W), weight seed, sharpness, image seed, EOS positions per image)
REFINE_CASES = [
    ("eos_s_refine_b5",    "parseq",             (32, 128), 76, 4.0, 86, [[7], [31], [32], [40, 55], []]),
    ("eos_base_refine_b5", "parseq-base-48x160", (48, 160), 77, 2.0, 87, [[3], [33], [63], [31, 45], []]),
]


REFINE_FP32_TOL = 5e-5      # reference fp32 against the fp64 oracle (the D = 768 sums are the longest)


def refine_context(nar_ids, bos_id, eos_positions):
    """[BOS, NAR argmax ids[:, :-1]] with every EOS replaced by id 1, then EOS (id 0) placed at the given positions."""
    ctx = torch.cat([torch.full_like(nar_ids[:, :1], bos_id), nar_ids[:, :-1]], dim=1).clone()
    ctx[:, 1:][ctx[:, 1:] == 0] = 1
    for b, pos in enumerate(eos_positions):
        for q in pos:
            ctx[b, q] = 0
    return ctx


def cloze_masks(ctx):
    """model.py:157,163: query i never sees key i + 1; every key from the first EOS on is padding."""
    L = ctx.shape[1]
    qmask = torch.zeros((L, L), dtype=torch.bool)
    qmask[torch.arange(L - 1), torch.arange(1, L)] = True
    pmask = (ctx == 0).int().cumsum(-1) > 0
    return qmask, pmask


def make_config_long(experiment: str, max_label_length: int, n_extra: int = 0, img_size=(32, 128), **kw):
    return make_config(experiment, charset_train=charset(n_extra), max_label_length=max_label_length,
                       img_size=tuple(img_size), **kw)


def _save(blob, name):
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    return size


def make_parseq():
    from oracle import reference_loader as RL
    from oracle.parseq_oracle import ParseqOracle
    for name, exp, mll, img, n_extra, wseed, B, iseed, ar, ri, ml in CASES:
        cfg = make_config_long(exp, mll, n_extra, img)
        sd = init_state_dict(cfg, wseed)
        ref, tok = RL.build_reference_model(cfg, sd)
        x = synth_images(cfg, B, iseed)
        ref.decode_ar, ref.refine_iters = ar, ri
        with torch.inference_mode():
            logits = ref(tok, x, ml).clone()
        o = ParseqOracle(cfg, sd, "fp64").forward(x, ml, ar, ri)
        assert o.logits.shape == logits.shape, (name, o.logits.shape, logits.shape)
        err = (o.logits.float() - logits).abs().max().item()
        assert err < 1e-5, (name, err)
        blob = dict(
            name=name, experiment=exp, max_label_length=mll, img_size=list(img), n_extra=n_extra, weight_seed=wseed,
            batch=B, image_seed=iseed, decode_ar=ar, refine_iters=ri, max_length=ml, sd_digest=state_dict_digest(sd),
            logits=logits.contiguous(), min_margin_fp64=o.min_margin.float(), steps=o.steps,
            ar_ids=None if o.ar_ids is None else o.ar_ids.int(),
            refine_ctx=[c.int() for c in o.refine_ctx],
            source="reference strhub.models.parseq.model.PARSeq (timm shim), torch %s CPU fp32" % torch.__version__,
        )
        size = _save(blob, name)
        print(f"{name:22s} L={mll + 1} C={cfg.num_classes} logits {tuple(logits.shape)} S={o.steps} "
              f"|ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


def make_vitstr():
    from oracle import reference_loader as RL
    from oracle.vitstr_oracle import VitstrOracle
    for name, mll, n_extra, wseed, B, iseed, ml in VITSTR_CASES:
        cfg = make_config_long("vitstr", mll, n_extra)
        sd = init_state_dict(cfg, wseed)
        ref = RL.build_reference_vitstr(cfg, sd)
        x = synth_images(cfg, B, iseed)
        m = cfg.max_label_length if ml is None else min(ml, cfg.max_label_length)
        with torch.inference_mode():
            logits = ref(x, m + 2)[:, 1:].clone()               # vitstr/system.py:67-70
        err = (VitstrOracle(cfg, sd, "fp64").system_forward(x, ml).float() - logits).abs().max().item()
        assert err < 1e-5, (name, err)
        blob = dict(name=name, experiment="vitstr", max_label_length=mll, img_size=list(cfg.img_size), n_extra=n_extra,
                    weight_seed=wseed, batch=B, image_seed=iseed, max_length=ml, sd_digest=state_dict_digest(sd),
                    logits=logits.contiguous(),
                    source="reference strhub.models.vitstr.model.ViTSTR (timm shim), torch %s CPU fp32" % torch.__version__)
        size = _save(blob, name)
        print(f"{name:22s} L={mll + 1} C={cfg.num_classes} logits {tuple(logits.shape)} |ref-fp64 oracle|={err:.2e} "
              f"{size / 1e6:.2f} MB")


def make_refine():
    from oracle import reference_loader as RL
    from oracle.parseq_oracle import ParseqOracle
    for name, exp, img, wseed, sharp, iseed, eos in REFINE_CASES:
        cfg = make_config_long(exp, 63, 0, img)
        sd = init_state_dict(cfg, wseed, sharp=sharp)
        ref, tok = RL.build_reference_model(cfg, sd)
        B, L = len(eos), 64
        x = synth_images(cfg, B, iseed)
        ref.decode_ar, ref.refine_iters = False, 0
        with torch.inference_mode():
            nar = ref(tok, x, 63)
            ctx = refine_context(nar.argmax(-1), tok.bos_id, eos)
            qmask, pmask = cloze_masks(ctx)
            # the refinement step of model.py:159-166 on the chosen context
            memory = ref.encode(x)
            pos_queries = ref.pos_queries[:, :L].expand(B, -1, -1)
            tgt_mask = torch.triu(torch.ones((L, L), dtype=torch.bool), 1)
            logits = ref.head(ref.decode(ctx, memory, tgt_mask, pmask, pos_queries, qmask)).clone()
        o = ParseqOracle(cfg, sd, "fp64")
        olog = o._decode(ctx, o.encode(x), o.p["pos_queries"][:, :L].expand(B, -1, -1), qmask, pmask).float()
        err = (olog - logits).abs().max().item()
        assert err < REFINE_FP32_TOL, (name, err)
        blob = dict(name=name, experiment=exp, max_label_length=63, img_size=list(img), n_extra=0, weight_seed=wseed,
                    sharp=sharp, batch=B, image_seed=iseed, decode_ar=False, refine_iters=1, max_length=63,
                    sd_digest=state_dict_digest(sd), eos_positions=eos, refine_ctx=[ctx.int()], logits=logits.contiguous(),
                    source="reference strhub.models.parseq.model.PARSeq (timm shim) refinement step on a given context, "
                           "torch %s CPU fp32" % torch.__version__)
        size = _save(blob, name)
        print(f"{name:22s} L={L} logits {tuple(logits.shape)} first EOS {[p[0] if p else None for p in eos]} "
              f"|ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    make_vitstr()
    make_parseq()
    make_refine()
