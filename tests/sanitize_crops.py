"""Tiny run of the raw-crop resize for compute-sanitizer (not a test):

    compute-sanitizer --tool memcheck python tests/sanitize_crops.py

One ragged batch with 1-pixel and 8192-pixel sides, the tall-crop pass order and a large crop, in every rotation, through
parseq_resize_crops, parseq_forward_crops and parseq_forward_host_crops (PARSeq-Ti, eager)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from parseq_b200.config import make_config
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict

SIZES = [(1, 1), (1, 8192), (8192, 1), (268, 2), (871, 1774), (33, 97), (128, 512)]

cfg = make_config("parseq-tiny")
m = create_model("parseq-tiny")
m.model.load_state_dict(init_state_dict(cfg, 0))
m.model.set_engine_option("use_graph", 0)
m = m.eval().to("cuda")
rng = np.random.default_rng(0)
crops = [torch.from_numpy(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)) for h, w in SIZES]
with torch.inference_mode():
    for r in (0, 90, 180, 270):
        u8 = m.preprocess([c.cuda() for c in crops], r)
        ld = m([c.cuda() for c in crops], rotation=r)
        lh = m(crops, rotation=r)
        torch.cuda.synchronize()
        assert torch.equal(ld.cpu(), lh)
print("sanitize_crops: ok", tuple(u8.shape))
