"""Generates tests/golden/orientation/*.pt: what the reference's own modules read from every crop of tests/golden/crops
(seeded and demo) in every orientation, and which orientation the search rule of tests/orientation_oracle.py picks by
the reference's `_eval_step` confidence.  Run where the reference tree exists:

    python tests/make_golden_orientation.py

Each crop is rotated and resized by the reference transform's CPU oracle (oracle/crop_transform.py, pinned to the
reference's own transform by tests/golden/crops), and read by strhub.models.parseq.model.PARSeq / the ViTSTR of
vitstr/model.py (under oracle/timm_shim.py) in fp64.  Per (orientation, crop) the golden keeps the ids through the first
EOS, the fp64 confidence (orientation_oracle.reference_confidence of the logits), the label length, and the smallest
top-1 - top-2 gap of every greedy decision that reaches the label (AR steps and each pass's rows through the EOS); per
crop the chosen orientation.  Weights are regenerated from (experiment, seed, classes) and verified by `sd_digest`:
sharp attention (q / k scaled) and a seeded head bias, as the other sharp goldens, so that the readings differ by
orientation and most decisions are clear of bf16 rounding.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

import crop_goldens                                                    # noqa: E402
import orientation_oracle as oo                                        # noqa: E402
from make_golden_long import make_config_long                          # noqa: E402
from oracle import crop_transform as ct                                # noqa: E402
from parseq_b200.weights import init_state_dict, state_dict_digest     # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "orientation")
GOLDEN_FILE_LIMIT = 1_000_000
ORIENTATIONS = (0, 90, 180, 270)
HEAD_BIAS_SIGMA = 3.0
# (case name, experiment, extra characters, weight seed, sharpness)
CASES = [
    ("or_s_sharp", "parseq", 0, 400, 4.0),
    ("or_ti_c3001", "parseq-tiny", 2906, 401, 4.0),
    ("or_vitstr_s", "vitstr", 0, 402, 0.0),
]


def state_dict(cfg, seed, sharp):
    """init_state_dict(cfg, seed, sharp) with head.bias = N(0, HEAD_BIAS_SIGMA) (seeded)."""
    sd = init_state_dict(cfg, seed, sharp=sharp)
    g = torch.Generator().manual_seed(seed + 7)
    sd["head.bias"] = (torch.randn(cfg.num_classes, generator=g, dtype=torch.float64) * HEAD_BIAS_SIGMA).to(torch.float32)
    return sd


def case_config(exp, n_extra):
    return make_config_long(exp, 25, n_extra)


def crops():
    """The seeded and demo crops of tests/golden/crops, in that order."""
    out = []
    for name in crop_goldens.NAMES:
        c, _ = crop_goldens.load(name)
        out += c
    return out


def _margins(heads, B):
    """Smallest top-1 - top-2 gap per image over the greedy decisions that reach its label."""
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
    return margin


def read(exp, cfg, sd, images):
    """fp64 reference logits [N, S, C] of float images [N, 3, H, W] and the margins of their decisions."""
    from oracle import reference_loader as RL
    x = images.double()
    heads = []
    if exp == "vitstr":
        ref = RL.build_reference_vitstr(cfg, sd).double()
        h = ref.head.register_forward_hook(lambda m, i, o: heads.append(o.detach()[:, 1:].clone()))
        with torch.no_grad():
            logits = ref(x, cfg.max_label_length + 2)[:, 1:].detach()      # vitstr/system.py:67-70
    else:
        ref, tok = RL.build_reference_model(cfg, sd)
        ref = ref.double()
        h = ref.head.register_forward_hook(lambda m, i, o: heads.append(o.detach().clone()))
        # with grad enabled nn.MultiheadAttention takes its reference path (see make_golden_attention.py)
        logits = ref(tok, x, None).detach()
    h.remove()
    return logits, _margins(heads, x.shape[0])


def make(case, cs):
    name, exp, n_extra, wseed, sharp = case
    cfg = case_config(exp, n_extra)
    sd = state_dict(cfg, wseed, sharp)
    N, L = len(cs), cfg.max_label_length + 1
    ids = torch.full((len(ORIENTATIONS), N, L), -1, dtype=torch.int16)
    conf = torch.zeros((len(ORIENTATIONS), N), dtype=torch.float64)
    length = torch.zeros((len(ORIENTATIONS), N), dtype=torch.int32)
    margin = torch.zeros((len(ORIENTATIONS), N), dtype=torch.float64)
    steps = []
    for k, r in enumerate(ORIENTATIONS):
        x = torch.from_numpy(np.stack([ct.transform(a, cfg.img_size, r) for a in cs]))
        logits, mg = read(exp, cfg, sd, x)
        steps.append(logits.shape[1])
        margin[k] = mg
        for b in range(N):
            c, n = oo.reference_confidence(logits[b].numpy())
            conf[k, b], length[k, b] = c, n
            row = logits[b].argmax(-1)[:min(n + 1, logits.shape[1])]
            ids[k, b, :row.numel()] = row.to(torch.int16)
    chosen, _ = oo.select(conf.T.numpy())
    blob = dict(name=name, experiment=exp, n_extra=n_extra, weight_seed=wseed, sharp=sharp,
                head_bias_sigma=HEAD_BIAS_SIGMA, sd_digest=state_dict_digest(sd), orientations=ORIENTATIONS,
                steps=steps, ids=ids, confidence=conf, length=length, min_margin=margin,
                chosen=torch.from_numpy(chosen),
                source="reference strhub.models.parseq.model.PARSeq / vitstr ViTSTR (timm shim) on the reference "
                       "transform of tests/golden/crops, fp64, torch %s CPU" % torch.__version__)
    path = os.path.join(OUT, name + ".pt")
    torch.save(blob, path)
    size = os.path.getsize(path)
    assert size < GOLDEN_FILE_LIMIT, (name, size)
    srt = conf.T.sort(dim=1, descending=True).values
    gap = (srt[:, 0] - srt[:, 1]) / srt[:, 0]
    clear = (margin.min(0).values > 2e-2) & (gap > 0.05)
    print(f"{name:12s} C={cfg.num_classes} steps={steps} chosen={chosen.tolist()} clear crops {int(clear.sum())}/{N} "
          f"{size / 1e3:.0f} KB")


if __name__ == "__main__":
    from oracle import reference_loader as RL
    assert RL.available(), "reference tree not present"
    os.makedirs(OUT, exist_ok=True)
    cs = crops()
    for case in CASES:
        make(case, cs)
