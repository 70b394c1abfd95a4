"""Tiny run of the orientation search for compute-sanitizer (not a test):

    compute-sanitizer --tool memcheck python tests/sanitize_orientation.py

Pass 1, the confidence kernel, pass 2 with padded readings and the select kernel at small sizes: PARSeq-Ti with
max_batch 5 (super-chunks of 5 // (R - 1) crops, readings rounded up to a power of two and capped at 5), every R, a
threshold, an allowlist, attention maps, refine_iters 0 (the zeroed tail rows), host crops and per-crop rotations; eager
and graph."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from parseq_b200.config import make_config
from parseq_b200.factory import create_model
from parseq_b200.weights import init_state_dict

cfg = make_config("parseq-tiny")
m = create_model("parseq-tiny")
m.model.load_state_dict(init_state_dict(cfg, 0))
m.model.set_engine_option("max_batch", 5)
m = m.eval().to("cuda")
rng = np.random.default_rng(0)
crops = [torch.from_numpy(rng.integers(0, 256, (int(rng.integers(1, 60)), int(rng.integers(1, 200)), 3), dtype=np.uint8))
         for _ in range(7)]
dev = [c.cuda() for c in crops]
with torch.inference_mode():
    for graph in (0, 1):
        m.model.set_engine_option("use_graph", graph)
        for o in ((0,), (180, 0), (0, 90, 270), (270, 180, 90, 0)):
            m.read_oriented(dev, o)
            m.read_oriented(crops, o, min_confidence=0.5, allowlist="0123456789abc")
            m.locate(dev, orientations=o)
        m.model.refine_iters = 0
        m.model.read_oriented(dev, (0, 90, 180, 270), attn_maps=True)
        m.model.refine_iters = 1
        m(dev, rotation=[0, 90, 180, 270, 0, 90, 180])
        torch.cuda.synchronize()
print("sanitize_orientation: ok")
