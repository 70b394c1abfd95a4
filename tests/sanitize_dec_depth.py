"""Tiny end-to-end run for compute-sanitizer (not a test):

    compute-sanitizer --tool memcheck python tests/sanitize_dec_depth.py

PARSeq-Ti decoders of depth 2 and 3: the content K/V cache writes of the AR steps (one row per image at pitch L), of the
NAR and refinement passes (whole contexts at pitch nkeys), of PARSeq.decode with a content mask, and of L = 64 (two keys
per lane)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.config import make_config
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict, synth_images

# (dec_depth, max_label_length, decode_ar, refine_iters, batch)
RUNS = [(2, 25, True, 1, 3), (3, 25, False, 2, 2), (2, 63, True, 1, 2)]

for depth, mll, ar, ri, B in RUNS:
    cfg = make_config("parseq-tiny", dec_depth=depth, max_label_length=mll)
    m = create_model("parseq-tiny", dec_depth=depth, max_label_length=mll, decode_ar=ar, refine_iters=ri)
    m.model.load_state_dict(init_state_dict(cfg, 0))
    m.model.set_engine_option("use_graph", 0)
    m = m.eval().to("cuda")
    x = synth_images(cfg, B, 1).cuda()
    with torch.inference_mode():
        out = m(x)
        mem = m.model.encode(x)
        J = 7
        tgt = torch.full((B, J), cfg.num_tokens - 2, dtype=torch.long, device="cuda")
        tgt[:, 1:] = 3
        cmask = torch.triu(torch.ones((J, J), dtype=torch.bool, device="cuda"), 1)
        dec = m.model.decode(tgt, mem, cmask)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(dec).all()
    print("ok: depth", depth, "L", mll + 1, "ar", ar, "refine", ri, "batch", B, tuple(out.shape), flush=True)
print("sanitize_dec_depth done")
