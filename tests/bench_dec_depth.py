"""Throughput and latency against the decoder depth (not a test):

    python tests/bench_dec_depth.py [--out FILE]

PARSeq-S, AR + 1 refinement, at 32x128 (max_label_length 25):
  * depth 1 on the cluster AR kernel (the default),
  * depth 1 with the AR loop on the chain of separate kernels (ar_kernel = 0), the path every deeper decoder runs,
  * depths 2 and 3 (chain),
each with device images/s at bs = 512 (CUDA-graph replay, CUDA events), the engine's per-category device time of one
bs = 512 forward in timing mode, and bs = 1 p50 latency (graph replay, host clock around a synchronised call).
Prints one JSON line per configuration with the card's name and power limit."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_label_length import card  # noqa: E402
import time  # noqa: E402

import torch  # noqa: E402

from parseq_b200.config import make_config  # noqa: E402
from parseq_b200.engine import Engine  # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images  # noqa: E402


def bench(depth, ar_kernel, iters, B=512):
    cfg = make_config("parseq", dec_depth=depth)
    sd = init_state_dict(cfg, 0)
    eng = Engine(cfg, 0, max_batch=B)
    st = torch.cuda.current_stream().cuda_stream
    eng.load_state_dict(sd, st)
    eng.set_option("ar_kernel", ar_kernel)
    x = synth_images(cfg, B, 1).cuda()
    L = eng.num_steps(None)
    logits = torch.empty((B, L, cfg.num_classes), device="cuda")
    ids = torch.empty((B, L), dtype=torch.int32, device="cuda")
    steps = torch.empty((1,), dtype=torch.int32, device="cuda")

    def fwd(n):
        eng.forward(x.data_ptr(), n, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, 25, True, 1)

    for _ in range(3):
        fwd(B)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fwd(B)
    b.record()
    torch.cuda.synchronize()
    dev_ms = a.elapsed_time(b) / iters
    eng.set_option("timing", 1)
    fwd(B)
    torch.cuda.synchronize()
    t = eng.get_timing()
    eng.set_option("timing", 0)
    lat = []
    for i in range(20 + 5 * iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fwd(1)
        torch.cuda.synchronize()
        if i >= 20:
            lat.append((time.perf_counter() - t0) * 1e3)
    lat.sort()
    eng.close()
    return dict(dec_depth=depth, ar_kernel=ar_kernel, batch=B, device_img_s=round(B / dev_ms * 1e3),
                device_ms=round(dev_ms, 3), category_ms={k: round(v["ms"], 3) for k, v in t.items()},
                bs1_p50_ms=round(lat[len(lat) // 2], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--configs", default="1:2,1:0,2:2,3:2", help="dec_depth:ar_kernel pairs")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = []
    for c in args.configs.split(","):
        depth, ak = (int(v) for v in c.split(":"))
        r = bench(depth, ak, args.iters)
        r["card"] = card()
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
