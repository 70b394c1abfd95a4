"""Throughput and latency against the size of the character set (not a test):

    python tests/bench_charset.py [--out FILE]

PARSeq-S, AR + 1 refinement, charset = 94_full + CJK ideographs, C in {94, 1000, 4000, 7000, 16384} head classes:
  * device images/s at bs = 512 (CUDA-graph replay, CUDA events),
  * the engine's per-category device time of one bs = 512 forward in timing mode (AR kernel, decoder GEMMs),
  * end-to-end images/s of the host-buffer entry point at bs = 512 (pinned host images in, [B, 26, C] fp32 logits out:
    26 * C * 4 bytes per image cross PCIe),
  * bs = 1 p50 latency (graph replay, host clock around a synchronised call).
Prints one JSON line per C and the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from parseq_b200.config import CHARSET_94, make_config  # noqa: E402
from parseq_b200.engine import Engine  # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def bench(C, iters, B=512):
    charset = CHARSET_94[: min(C - 1, 94)] + "".join(chr(0x4E00 + i) for i in range(max(0, C - 1 - 94)))
    cfg = make_config("parseq", charset_train=charset)
    assert cfg.num_classes == C
    sd = init_state_dict(cfg, 0)
    eng = Engine(cfg, 0, max_batch=B)
    st = torch.cuda.current_stream().cuda_stream
    eng.load_state_dict(sd, st)
    x = synth_images(cfg, B, 1).cuda()
    L = eng.num_steps(None)
    logits = torch.empty((B, L, C), device="cuda")
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
    # host buffers: pinned images in, pinned logits / ids out
    xh = x.cpu().pin_memory()
    lh = torch.empty((B, L, C), pin_memory=True)
    ih = torch.empty((B, L), dtype=torch.int32, pin_memory=True)
    sh = torch.empty((1,), dtype=torch.int32, pin_memory=True)
    for _ in range(2):
        eng.forward_host(xh.data_ptr(), B, lh.data_ptr(), ih.data_ptr(), sh.data_ptr(), st, 25, True, 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        eng.forward_host(xh.data_ptr(), B, lh.data_ptr(), ih.data_ptr(), sh.data_ptr(), st, 25, True, 1)
    torch.cuda.synchronize()
    host_s = (time.perf_counter() - t0) / iters
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
    return dict(C=C, batch=B, device_img_s=round(B / dev_ms * 1e3), device_ms=round(dev_ms, 3),
                ar_kernel_ms=round(t["dec_ar"]["ms"], 3), dec_gemm_ms=round(t["dec_gemm"]["ms"], 3),
                host_img_s=round(B / host_s), logits_bytes_per_img=26 * C * 4, bs1_p50_ms=round(lat[len(lat) // 2], 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--classes", default="94,1000,4000,7000,16384")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = []
    for C in (int(c) for c in args.classes.split(",")):
        r = bench(C, args.iters)
        r["card"] = card()
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
