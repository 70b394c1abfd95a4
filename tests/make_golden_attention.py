"""Generates tests/golden/attention/*.pt: cross-attention maps computed by the reference's own modules
(strhub.models.parseq.model.PARSeq under oracle/timm_shim.py) in fp64.  Run where the reference tree exists:

    python tests/make_golden_attention.py

A forward hook on decoder.layers[-1].cross_attn records output[1] of every call: nn.MultiheadAttention's head-averaged
ca_weights of the last layer's query stream (modules.py:74).  Each AR step contributes its one row, each NAR or cloze
pass all of its rows; the maps of parseq_forward_args.attn_maps are those of the pass that produced the returned logits
(the last refinement pass, the NAR pass, or the AR steps, S of them after a batch-wide early exit).  A forward hook on
the head records every logits row the model decided on, so each image's smallest top-1 / top-2 margin over all its
greedy decisions is stored with it: where that margin clears the engine's bf16 error, its ids are the reference's.

The weights are the seeded synthetic ones of parseq_b200.weights (sharp attention where asked) with a seeded head bias
(sigma 3, EOS level with the second-best class): a random head is nearly flat, so no decision would be clear, and the bias ends
most readings within a few characters.  With an allowlist the head is wrapped as tests/make_golden_allowlist.py wraps
it (every other class -inf).  Each golden holds ids, maps, margins, steps and what regenerates weights, images and
allowlists (`sd_digest` checks them).
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

OUT = os.path.join(ROOT, "tests", "golden", "attention")
GOLDEN_FILE_LIMIT = 1_000_000
HEAD_BIAS_SIGMA = 3.0
DIGITS = "0123456789"

# (case name, experiment, dec_depth, max_label_length, extra characters, weight seed, sharpness, batch, image seed,
#  decode_ar, refine_iters, max_length, allowlist or None)
CASES = [
    ("am_s_ar1_b3",        "parseq",             1, 25, 0,    300, 4.0, 3, 310, True,  1, None, None),
    ("am_s_ar0_exit_b3",   "parseq",             1, 25, 0,    301, 4.0, 3, 311, True,  0, None, None),
    ("am_s_nar0_b2",       "parseq",             1, 25, 0,    302, 4.0, 2, 312, False, 0, None, None),
    ("am_s_nar2_b2",       "parseq",             1, 25, 0,    303, 4.0, 2, 313, False, 2, None, None),
    ("am_ti_ar1_b3",       "parseq-tiny",        1, 25, 0,    304, 4.0, 3, 314, True,  1, None, None),
    ("am_p16_ar1_b2",      "parseq-patch16-224", 1, 25, 0,    305, 4.0, 2, 315, True,  1, None, None),
    ("am_s_l64_ar1_b2",    "parseq",             1, 63, 0,    306, 4.0, 2, 316, True,  1, None, None),
    ("am_d2_s_ar1_b2",     "parseq",             2, 25, 0,    307, 2.0, 2, 317, True,  1, 25,   None),
    ("am_ti_c3001_ar1_b3", "parseq-tiny",        1, 25, 2906, 308, 4.0, 3, 318, True,  1, None,
     [DIGITS, None, "abc" + "".join(chr(0x4E00 + i) for i in range(0, 2906, 97))]),
]

# EOS bias of the early-exit case: every image emits EOS within a few steps, so the AR loop stops at S < L
EOS_BIAS = {"am_s_ar0_exit_b3": 0.6}


def golden_state_dict(cfg, seed, sharp, eos=0.0):
    """init_state_dict(cfg, seed, sharp) with head.bias = N(0, HEAD_BIAS_SIGMA) (seeded) and EOS at the second-best
    class's bias + eos (the best class's at eos = 1: a batch-wide early exit)."""
    sd = init_state_dict(cfg, seed, sharp=sharp)
    g = torch.Generator().manual_seed(seed + 7)
    bias = torch.randn(cfg.num_classes, generator=g, dtype=torch.float64) * HEAD_BIAS_SIGMA
    top = bias[1:].topk(2).values
    bias[0] = top[1] + eos * (top[0] - top[1])
    sd["head.bias"] = bias.to(torch.float32)
    return sd


def make(case):
    from allowlist_oracle import MaskedHead, allowed_from_strings
    from oracle import reference_loader as RL
    name, exp, depth, mll, n_extra, wseed, sharp, B, iseed, ar, ri, ml, allowlist = case
    img = (224, 224) if exp == "parseq-patch16-224" else (32, 128)
    cfg = make_config_long(exp, mll, n_extra, img_size=img, dec_depth=depth)
    eos = EOS_BIAS.get(name, 0.0)
    sd = golden_state_dict(cfg, wseed, sharp, eos)
    ref, tok = RL.build_reference_model(cfg, sd)
    ref = ref.double()
    ref.decode_ar, ref.refine_iters = ar, ri
    if allowlist is not None:
        ref.head = MaskedHead(ref.head, allowed_from_strings(tok, allowlist, cfg.num_classes))
    x = synth_images(cfg, B, iseed).double()
    calls, heads = [], []
    h1 = ref.decoder.layers[-1].cross_attn.register_forward_hook(lambda m, i, o: calls.append(o[1].detach().clone()))
    h2 = ref.head.register_forward_hook(lambda m, i, o: heads.append(o.detach().clone()))
    # with grad enabled (the parameters require it) nn.MultiheadAttention takes its reference path, not the fused
    # inference fast path, whose mask merging rejects the AR steps' sliced masks
    logits = ref(tok, x, ml).detach()
    h1.remove()
    h2.remove()
    S = logits.shape[1]
    assert name != "am_s_ar0_exit_b3" or S < mll + 1, (name, S)
    maps = calls[-1] if ri or not ar else torch.cat(calls[:S], dim=1)
    assert maps.shape == (B, S, cfg.num_patches), (name, maps.shape)
    # every greedy decision that reaches a label: the AR steps of an image until it emits EOS, and each pass's rows up
    # to its first EOS (later context tokens are masked by the padding mask, later ids are not part of the label)
    margin = torch.full((B,), float("inf"), dtype=torch.float64)
    done = torch.zeros(B, dtype=torch.bool)
    for h in heads:
        h = h.reshape(B, -1, h.shape[-1])
        top2 = h.topk(2, dim=-1).values
        gap = top2[..., 0] - top2[..., 1]
        arg = h.argmax(-1)
        if h.shape[1] == 1:                        # one AR step
            gap = torch.where(done, torch.inf, gap[:, 0])
            done |= arg[:, 0] == 0
        else:
            seen = (arg == 0).int().cumsum(-1)
            live = (seen == 0) | ((seen == 1) & (arg == 0))
            gap = torch.where(live, gap, torch.inf).min(dim=1).values
        margin = torch.minimum(margin, gap)
    ids = logits.argmax(-1)
    blob = dict(name=name, experiment=exp, dec_depth=depth, max_label_length=mll, n_extra=n_extra, weight_seed=wseed,
                sharp=sharp, eos_bias=eos, batch=B, image_seed=iseed, decode_ar=ar, refine_iters=ri, max_length=ml,
                allowlist=allowlist,
                sd_digest=state_dict_digest(sd), steps=S, ids=ids.int(), maps=maps.contiguous(), min_margin=margin,
                source="reference strhub.models.parseq.model.PARSeq (timm shim), forward hook on "
                       "decoder.layers[-1].cross_attn, fp64, torch %s CPU" % torch.__version__)
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    print(f"{name:20s} C={cfg.num_classes} T={cfg.num_patches} S={S} maps {tuple(maps.shape)} "
          f"margins {[round(v, 3) for v in margin.tolist()]} {size / 1e3:.0f} KB")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    for case in CASES:
        make(case)
