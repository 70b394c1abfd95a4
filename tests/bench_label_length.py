"""Throughput and latency against the label length (not a test):

    python tests/bench_label_length.py [--out FILE]

PARSeq-S, AR + 1 refinement, 94_full charset, at 32x128 with max_label_length 25, 31, 47, 63 (L = 26, 32, 48, 64 decode
positions) and at 32x256 with max_label_length 63:
  * device images/s at bs = 512 (CUDA-graph replay, CUDA events),
  * the engine's per-category device time of one bs = 512 forward in timing mode (AR kernel, decoder GEMMs),
  * bs = 1 p50 latency (graph replay, host clock around a synchronised call).
Prints one JSON line per configuration with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from parseq_b200.config import make_config  # noqa: E402
from parseq_b200.engine import Engine  # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def bench(mll, img_w, iters, B=512):
    cfg = make_config("parseq", max_label_length=mll, img_size=(32, img_w))
    sd = init_state_dict(cfg, 0)
    eng = Engine(cfg, 0, max_batch=B)
    st = torch.cuda.current_stream().cuda_stream
    eng.load_state_dict(sd, st)
    x = synth_images(cfg, B, 1).cuda()
    L = eng.num_steps(None)
    C = cfg.num_classes
    logits = torch.empty((B, L, C), device="cuda")
    ids = torch.empty((B, L), dtype=torch.int32, device="cuda")
    steps = torch.empty((1,), dtype=torch.int32, device="cuda")

    def fwd(n):
        eng.forward(x.data_ptr(), n, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, mll, True, 1)

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
    return dict(img=f"32x{img_w}", max_label_length=mll, L=L, batch=B, device_img_s=round(B / dev_ms * 1e3),
                device_ms=round(dev_ms, 3), ar_kernel_ms=round(t["dec_ar"]["ms"], 3),
                dec_gemm_ms=round(t["dec_gemm"]["ms"], 3), bs1_p50_ms=round(lat[len(lat) // 2], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--configs", default="25:128,31:128,47:128,63:128,63:256",
                    help="max_label_length:image width pairs")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = []
    for c in args.configs.split(","):
        mll, w = (int(v) for v in c.split(":"))
        r = bench(mll, w, args.iters)
        r["card"] = card()
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
