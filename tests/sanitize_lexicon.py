"""Tiny run of lexicon-constrained beam search for compute-sanitizer (not a test):

    compute-sanitizer --tool memcheck python tests/sanitize_lexicon.py

PARSeq-Ti with 1 and 2 decoder layers at 95 and 3001 classes and ViTSTR-S, max_label_length 63: beam widths 1, 5 and
16, groups of one image at K = 16 (dec_chunk = 16), two super-chunks (max_batch = 16), a shared lexicon with "" and
words of 63 characters, per-image lexicons, an allowlist, uint8 input and max_length."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import numpy as np
import torch
from make_golden_long import charset, make_config_long
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict, synth_images

rng = np.random.default_rng(0)
for exp, depth, n_extra in (("parseq-tiny", 1, 0), ("parseq-tiny", 2, 0), ("parseq-tiny", 1, 2906), ("vitstr", 1, 0)):
    cs = charset(n_extra)
    r = random.Random(1)
    words = ["", cs[:1], cs[:2], cs[-1] * 63] + ["".join(r.choice(cs) for _ in range(r.randint(1, 12))) for _ in range(300)]
    per = [words[i * 10:(i + 1) * 10] + [""] for i in range(20)]
    extra = {} if exp == "vitstr" else {"dec_depth": depth}
    cfg = make_config_long(exp, 63, n_extra, **extra)
    m = create_model(exp, charset_train=cs, max_label_length=63, **extra)
    (m if exp == "vitstr" else m.model).load_state_dict(init_state_dict(cfg, 0))
    m.model.set_engine_option("max_batch", 16)
    m.model.set_engine_option("dec_chunk", 16)
    m = m.eval().to("cuda")
    x = synth_images(cfg, 20, 1).cuda()
    with torch.inference_mode():
        for K in (1, 5, 16):
            labels, scores = m.beam_search(x, K, lexicon=words, allowlist=[None, "abc", "", None, cs[:20]] * 4)
            m.beam_search(x, K, lexicon=per)
        u8 = torch.from_numpy(rng.integers(0, 256, (20, *cfg.img_size, 3), dtype=np.uint8)).cuda()
        m.beam_search(u8, 3, max_length=7, lexicon=words)
    torch.cuda.synchronize()
    print(exp, depth, n_extra, tuple(scores.shape), [len(h) for h in labels])
print("sanitize_lexicon: ok")
