"""Tiny run of the region warp for compute-sanitizer (not a test):

    compute-sanitizer --tool memcheck python tests/sanitize_regions.py

The golden regions (1 x 1 and 1 x N crops, an 8192-wide crop, regions partly and wholly outside their frame, a 1 x 1
frame and a 6000 x 4000 frame) through parseq_warp_regions in one call and in chunks of max_batch = 16, then
forward on the crops (PARSeq-Ti, eager)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

import make_golden_regions as mg  # noqa: E402
from parseq_b200.config import make_config  # noqa: E402
from parseq_b200.factory import create_model  # noqa: E402
from parseq_b200.weights import init_state_dict  # noqa: E402

cfg = make_config("parseq-tiny")
m = create_model("parseq-tiny")
m.model.load_state_dict(init_state_dict(cfg, 0))
m.model.set_engine_option("use_graph", 0)
m = m.eval().to("cuda")
frames, g = mg.load()
dev = [torch.from_numpy(f).cuda() for f in frames]
with torch.inference_mode():
    rc = m.crop_regions(dev, g["quads"], frame_index=g["frame_index"])
    m.model.set_engine_option("max_batch", 16)
    rc16 = m.crop_regions(dev, g["quads"], frame_index=g["frame_index"])
    logits = m(rc16)
    torch.cuda.synchronize()
assert [mg.digest(c.cpu().numpy()) for c in rc] == g["sha256"]
assert all(torch.equal(a, b) for a, b in zip(rc, rc16))
print("sanitize_regions: ok", len(rc), tuple(logits.shape))
