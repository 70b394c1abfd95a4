"""Generates tests/golden/allowlist/*.pt: golden outputs of the reference's own modules (strhub.models.parseq.model.PARSeq
and strhub.models.vitstr.model.ViTSTR under oracle/timm_shim.py) with the character head wrapped by a per-image allowlist
(tests/allowlist_oracle.py MaskedHead: disallowed classes -> -inf).  Run where the reference tree exists:

    python tests/make_golden_allowlist.py

Every golden is checked against the fp64 oracle with the same mask; `min_margin_fp64` is the smallest top-1 - top-2
gap over the allowed classes of every greedy decision an image took.  Weights are regenerated from (experiment, seed,
geometry) by parseq_b200.weights.init_state_dict and verified through `sd_digest`.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

from make_golden_long import charset, make_config_long                 # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images, state_dict_digest  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "allowlist")
GOLDEN_FILE_LIMIT = 1_000_000
DIGITS = "0123456789"
# one allowlist per image: a digits-only field, mixed per-image sets, an empty allowlist, an unconstrained image
MIXED = [DIGITS, "abcdefghijklmnopqrstuvwxyz", DIGITS + "-/.", "", None, "ABCDEF0123456789", DIGITS, "0123456789.,$"]
# single characters: with EOS two candidates per decision, so that images whose every decision is clear of bf16
# rounding (min_margin_fp64 > 2e-2 over the allowed classes) remain for the bit-exact id comparison on the GPU
SINGLE = ["7", "a", "Z", "3", "q", "%", "5", "x", "K", "0", "m", "?", "8", "b", "T", "2"]
WIDE = "WIDE"                    # the allowlist is derived from the unconstrained run (see wide_allowlist)

# (case name, experiment, dec_depth, max_label_length, extra characters, weight seed, batch, image seed, decode_ar,
#  refine_iters, max_length, allowlist)
CASES = [
    ("al_s_ar1_b16",       "parseq",      1, 25, 0,    120, 16, 130, True,  1, None, MIXED + SINGLE[:8]),
    ("al_ti_nar2_b12",     "parseq-tiny", 1, 25, 0,    121, 12, 131, False, 2, None, MIXED[:4] + SINGLE[:8]),
    ("al_s_ar0_b12",       "parseq",      1, 25, 0,    122, 12, 132, True,  0, None, [DIGITS, None, "abc"] + SINGLE[:9]),
    ("al_ti_c3001_ar1_b4", "parseq-tiny", 1, 25, 2906, 123, 4,  133, True,  1, 10,   WIDE),
    ("al_d2_s_ar1_b12",    "parseq",      2, 25, 0,    124, 12, 134, True,  1, None, MIXED[:3] + SINGLE[:9]),
    ("al_s_l64_ar0_b16",   "parseq",      1, 63, 0,    125, 16, 135, True,  0, None, [DIGITS, None, "xyz0123"] + SINGLE[:13]),
]
# (case name, max_label_length, weight seed, batch, image seed, max_length, allowlist)
VITSTR_CASES = [
    ("al_vitstr_s_b4", 25, 126, 4, 136, None, [DIGITS, "", None, "abcdef"]),
]


def wide_allowlist(cs: str, free_ids: torch.Tensor, seed: int):
    """Per image: one seeded character of the class-sliced head's far slices that the unconstrained model never picked,
    so that the mask overrules the unconstrained argmax at every step where that was not EOS."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for row in free_ids:
        banned = {int(i) for i in row.tolist()}
        while True:
            i = int(torch.randint(1000, len(cs) + 1, (), generator=g))
            if i not in banned:
                out.append(cs[i - 1])
                break
    return out


def _save(blob, name):
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    return size


def _check(ref_logits, oracle_logits, name):
    inf_ref, inf_or = torch.isneginf(ref_logits), torch.isneginf(oracle_logits)
    assert torch.equal(inf_ref, inf_or), name
    err = (oracle_logits.float() - ref_logits)[~inf_ref].abs().max().item()
    assert err < 1e-5, (name, err)
    return err


def make_parseq():
    from allowlist_oracle import MaskedHead, allowed_from_strings, masked_oracle
    from dec_depth_oracle import DepthOracle
    from oracle import reference_loader as RL
    from oracle.parseq_oracle import ParseqOracle
    for name, exp, depth, mll, n_extra, wseed, B, iseed, ar, ri, ml, allowlist in CASES:
        cfg = make_config_long(exp, mll, n_extra, dec_depth=depth)
        sd = init_state_dict(cfg, wseed)
        ref, tok = RL.build_reference_model(cfg, sd)
        x = synth_images(cfg, B, iseed)
        ref.decode_ar, ref.refine_iters = ar, ri
        if allowlist == WIDE:
            with torch.inference_mode():
                free = ref(tok, x, ml).argmax(-1)
            allowlist = wide_allowlist(charset(n_extra), free, wseed)
        allowed = allowed_from_strings(tok, allowlist, cfg.num_classes)
        head = ref.head
        ref.head = MaskedHead(head, allowed)
        with torch.inference_mode():
            logits = ref(tok, x, ml).clone()
        ref.head = head
        o = masked_oracle(DepthOracle if depth > 1 else ParseqOracle)(cfg, sd, "fp64")
        o.allowed = allowed
        out = o.forward(x, ml, ar, ri)
        assert out.logits.shape == logits.shape, (name, out.logits.shape, logits.shape)
        err = _check(logits, out.logits, name)
        ids = logits.argmax(-1)
        for b, s in enumerate(allowlist):
            assert bool(allowed[b][ids[b]].all()), name
        blob = dict(
            name=name, experiment=exp, dec_depth=depth, max_label_length=mll, img_size=list(cfg.img_size), n_extra=n_extra,
            weight_seed=wseed, batch=B, image_seed=iseed, decode_ar=ar, refine_iters=ri, max_length=ml,
            sd_digest=state_dict_digest(sd), allowlist=list(allowlist), logits=logits.contiguous(), ids=ids.int(),
            min_margin_fp64=out.min_margin.float(), steps=out.steps,
            ar_ids=None if out.ar_ids is None else out.ar_ids.int(), refine_ctx=[c.int() for c in out.refine_ctx],
            source="reference strhub.models.parseq.model.PARSeq (timm shim) with a per-image masked head, torch %s CPU "
                   "fp32" % torch.__version__,
        )
        size = _save(blob, name)
        print(f"{name:20s} C={cfg.num_classes} logits {tuple(logits.shape)} S={out.steps} margins "
              f"{[round(v, 3) for v in out.min_margin.tolist()]} |ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


def make_vitstr():
    from allowlist_oracle import MaskedHead, MaskedVitstrOracle, allowed_from_strings
    from oracle import reference_loader as RL
    from parseq_b200.tokenizer import Tokenizer
    for name, mll, wseed, B, iseed, ml, allowlist in VITSTR_CASES:
        cfg = make_config_long("vitstr", mll, 0)
        sd = init_state_dict(cfg, wseed)
        ref = RL.build_reference_vitstr(cfg, sd)
        allowed = allowed_from_strings(Tokenizer(cfg.charset_train), allowlist, cfg.num_classes)
        ref.head = MaskedHead(ref.head, allowed)
        x = synth_images(cfg, B, iseed)
        m = cfg.max_label_length if ml is None else min(ml, cfg.max_label_length)
        with torch.inference_mode():
            logits = ref(x, m + 2)[:, 1:].clone()               # vitstr/system.py:67-70
        o = MaskedVitstrOracle(cfg, sd, "fp64")
        o.allowed = allowed
        ol = o.system_forward(x, ml)
        err = _check(logits, ol, name)
        top2 = ol.topk(2, dim=-1).values
        margin = torch.where(torch.isneginf(top2[..., 1]), torch.full_like(top2[..., 0], float("inf")),
                             top2[..., 0] - top2[..., 1]).min(dim=-1).values
        blob = dict(name=name, experiment="vitstr", dec_depth=1, max_label_length=mll, img_size=list(cfg.img_size),
                    n_extra=0, weight_seed=wseed, batch=B, image_seed=iseed, max_length=ml, sd_digest=state_dict_digest(sd),
                    allowlist=list(allowlist), logits=logits.contiguous(), ids=logits.argmax(-1).int(),
                    min_margin_fp64=margin.float(),
                    source="reference strhub.models.vitstr.model.ViTSTR (timm shim) with a per-image masked head, "
                           "torch %s CPU fp32" % torch.__version__)
        size = _save(blob, name)
        print(f"{name:20s} logits {tuple(logits.shape)} margins {[round(v, 3) for v in margin.tolist()]} "
              f"|ref-fp64 oracle|={err:.2e} {size / 1e6:.2f} MB")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    make_vitstr()
    make_parseq()
