"""Tiny run of candidate scoring for compute-sanitizer (not a test):

    compute-sanitizer --tool memcheck python tests/sanitize_score.py

PARSeq-Ti with 1 and 2 decoder layers and ViTSTR-S at max_label_length 63: ragged candidates of 0 to 63 characters,
groups split inside an image (dec_chunk = 2), two super-chunks (max_batch = 4), float and uint8 inputs, per-position
terms on."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from make_golden_long import charset, make_config_long
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict, synth_images

rng = np.random.default_rng(0)
cs = charset(0)
for exp, depth in (("parseq-tiny", 1), ("parseq-tiny", 2), ("vitstr", 1)):
    extra = {} if exp == "vitstr" else {"dec_depth": depth}
    cfg = make_config_long(exp, 63, 0, **extra)
    m = create_model(exp, charset_train=cs, max_label_length=63, **extra)
    (m if exp == "vitstr" else m.model).load_state_dict(init_state_dict(cfg, 0))
    m.model.set_engine_option("max_batch", 4)
    m.model.set_engine_option("dec_chunk", 2)
    m = m.eval().to("cuda")
    x = synth_images(cfg, 6, 1).cuda()
    cands = [["".join(cs[i] for i in rng.integers(0, 94, n)) for n in rng.integers(0, 64, 1 + b % 4)] + [""] for b in range(6)]
    with torch.inference_mode():
        s, t = m.score(x, cands, return_token_logprobs=True)
        u8 = torch.from_numpy(rng.integers(0, 256, (6, *cfg.img_size, 3), dtype=np.uint8)).cuda()
        m.score(u8, cands)
    torch.cuda.synchronize()
    print(exp, depth, tuple(s.shape), bool(torch.isfinite(s[s > -float("inf")]).all()))
print("sanitize_score: ok")
