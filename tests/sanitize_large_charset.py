"""Tiny end-to-end run for compute-sanitizer (not a test):

    compute-sanitizer --tool racecheck|synccheck|memcheck python tests/sanitize_large_charset.py

PARSeq-Ti and -S with 300 head classes: the cluster AR kernel's class-sliced head (a TMA stream of the CTA's head slice,
logits stored from the fragments, one (max, index) pair per row exchanged through distributed shared memory and merged
after an extra cluster barrier) in both cluster sizes, its head-split variant (one image) and the chain path."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.config import CHARSET_94, make_config
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict, synth_images

CHARSET = CHARSET_94 + "".join(chr(0x4E00 + i) for i in range(205))     # 300 head classes
# (ar_kernel, ar_cluster_size, batch)
RUNS = [(2, 8, 1), (2, 8, 19), (2, 6, 19), (0, 0, 3)]

for exp in ("parseq-tiny", "parseq"):
    cfg = make_config(exp, charset_train=CHARSET)
    sd = init_state_dict(cfg, 0)
    for impl, cs, B in RUNS:
        m = create_model(exp, charset_train=CHARSET, decode_ar=True, refine_iters=1)
        m.model.load_state_dict(sd)
        m.model.set_engine_option("use_graph", 0)
        m.model.set_engine_option("ar_kernel", impl)
        m.model.set_engine_option("ar_cluster_size", cs)
        m = m.eval().to("cuda")
        x = synth_images(cfg, B, 1).cuda()
        with torch.inference_mode():
            out = m(x, 6)
        torch.cuda.synchronize()
        assert torch.isfinite(out).all() and out.shape[-1] == 300
        print("ok:", exp, "ar_kernel", impl, "cluster", cs, "batch", B, tuple(out.shape), flush=True)
print("sanitize_large_charset done")
