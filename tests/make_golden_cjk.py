"""Generates tests/golden/cjk/*.pt: golden outputs of the reference's own modules (strhub.models.parseq.model.PARSeq and
strhub.models.vitstr.model.ViTSTR under oracle/timm_shim.py) for models with a large character set, plus the reference
Tokenizer over that charset.  Run where the reference tree exists:

    python tests/make_golden_cjk.py

The charset is synthetic: the 94 characters of 94_full followed by CJK ideographs chr(0x4E00 + i).  Weights are not
stored: they are regenerated from (experiment, seed, charset size) by parseq_b200.weights.init_state_dict and verified
through `sd_digest`.  The goldens live in a subdirectory of their own: the PARSeq and ViTSTR parity tests glob the files
at the top of tests/golden and build 94-character models for them.
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

OUT = os.path.join(ROOT, "tests", "golden", "cjk")
GOLDEN_FILE_LIMIT = 1_000_000


def cjk_charset(n_cjk: int) -> str:
    return CHARSET_94 + "".join(chr(0x4E00 + i) for i in range(n_cjk))


# (case name, experiment, CJK characters, weight seed, batch, image seed, decode_ar, refine_iters, max_length)
# head classes C = 94 + n_cjk + 1
CASES = [
    ("cjk_s_ar1_b2",       "parseq",      2906, 40, 2, 50, True,  1, None),   # C = 3001
    ("cjk_ti_nar2_b1",     "parseq-tiny", 4905, 41, 1, 51, False, 2, None),   # C = 5000
    ("cjk_ti_ar0_len5_b2", "parseq-tiny", 6905, 42, 2, 52, True,  0, 5),      # C = 7000
]
# (case name, CJK characters, weight seed, batch, image seed, max_length)
VITSTR_CASES = [
    ("cjk_vitstr_s_b1", 3905, 43, 1, 53, None),                                # C = 4000
]
TOKENIZER_CJK = 2906


def make_config_cjk(experiment: str, n_cjk: int, **kw):
    return make_config(experiment, charset_train=cjk_charset(n_cjk), **kw)


def _save(blob, name):
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    return size


def make_parseq():
    from oracle import reference_loader as RL
    from oracle.parseq_oracle import ParseqOracle
    for name, exp, n_cjk, wseed, B, iseed, ar, ri, ml in CASES:
        cfg = make_config_cjk(exp, n_cjk)
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
            name=name, experiment=exp, n_cjk=n_cjk, weight_seed=wseed, batch=B, image_seed=iseed,
            decode_ar=ar, refine_iters=ri, max_length=ml, sd_digest=state_dict_digest(sd),
            logits=logits.contiguous(), min_margin_fp64=o.min_margin.float(), steps=o.steps,
            ar_ids=None if o.ar_ids is None else o.ar_ids.int(),
            refine_ctx=[c.int() for c in o.refine_ctx],
            source="reference strhub.models.parseq.model.PARSeq (timm shim), torch %s CPU fp32" % torch.__version__,
        )
        size = _save(blob, name)
        print(f"{name:20s} C={cfg.num_classes} logits {tuple(logits.shape)} S={o.steps} |ref-fp64 oracle|={err:.2e} "
              f"{size / 1e6:.2f} MB")


def make_vitstr():
    from oracle import reference_loader as RL
    from oracle.vitstr_oracle import VitstrOracle
    for name, n_cjk, wseed, B, iseed, ml in VITSTR_CASES:
        cfg = make_config_cjk("vitstr", n_cjk)
        sd = init_state_dict(cfg, wseed)
        ref = RL.build_reference_vitstr(cfg, sd)
        x = synth_images(cfg, B, iseed)
        m = cfg.max_label_length if ml is None else min(ml, cfg.max_label_length)
        with torch.inference_mode():
            logits = ref(x, m + 2)[:, 1:].clone()               # vitstr/system.py:67-70
        err = (VitstrOracle(cfg, sd, "fp64").system_forward(x, ml).float() - logits).abs().max().item()
        assert err < 1e-5, (name, err)
        blob = dict(name=name, experiment="vitstr", n_cjk=n_cjk, weight_seed=wseed, batch=B, image_seed=iseed,
                    max_length=ml, sd_digest=state_dict_digest(sd), logits=logits.contiguous(),
                    source="reference strhub.models.vitstr.model.ViTSTR (timm shim), torch %s CPU fp32" % torch.__version__)
        size = _save(blob, name)
        print(f"{name:20s} C={cfg.num_classes} logits {tuple(logits.shape)} |ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


def make_tokenizer():
    from oracle import reference_loader as RL
    _, RefTok = RL.load_reference_classes()
    charset = cjk_charset(TOKENIZER_CJK)
    rt = RefTok(charset)
    C = len(charset) + 1
    labels_in = ["ab", "一丁z", cjk_charset(TOKENIZER_CJK)[-3:] + "!"]
    # decode: one row with an EOS inside, one running to the end; ids on both sides of the 94-character block
    seq = [[11, 95, 0, 13, 14], [C - 1, 96, 2, 500, C - 2]]
    probs = torch.zeros(2, 5, C)
    for b in range(2):
        for i, t in enumerate(seq[b]):
            probs[b, i, t] = 0.9
    labels, ps = rt.decode(probs)
    blob = dict(n_cjk=TOKENIZER_CJK, encode_labels=labels_in, encode=rt.encode(labels_in), decode_ids=torch.tensor(seq),
                decode_labels=labels, decode_label_probs=[p.clone() for p in ps])
    size = _save(blob, "cjk_tokenizer")
    print(f"cjk_tokenizer C={C} labels {labels} {size / 1e6:.2f} MB")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    make_tokenizer()
    make_vitstr()
    make_parseq()
