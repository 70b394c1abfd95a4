"""Cost of per-image character allowlists (not a test):

    python tests/bench_allowlist.py [--iters N] [--out FILE]

PARSeq-S, AR + 1 refinement, at C = 95 (94_full + EOS: the cluster kernel's redundant head) and C = 16384 (94_full + CJK:
its class-sliced head), for four masks: none (NULL), all ones, digits only, and per-image mixed sets:
  * device images/s at bs = 512 (CUDA-graph replay, CUDA events),
  * the AR kernel's device time of one bs = 512 forward in timing mode,
  * bs = 1 p50 latency (graph replay, host clock around a synchronised call).
Prints one JSON line per (C, mask) and the card's name and power limit."""
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
from parseq_b200.system import allowlist_mask  # noqa: E402
from parseq_b200.tokenizer import Tokenizer  # noqa: E402
from parseq_b200.weights import init_state_dict, synth_images  # noqa: E402

MIXED = ["0123456789", "0123456789-/.", "abcdefghijklmnopqrstuvwxyz", "ABCDEFGHJKLMNPRSTUVWXYZ0123456789", None]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def masks(charset, B, C):
    tok = Tokenizer(charset)
    return {"none": None, "ones": allowlist_mask(tok, charset, B, C), "digits": allowlist_mask(tok, "0123456789", B, C),
            "mixed": allowlist_mask(tok, [MIXED[b % len(MIXED)] for b in range(B)], B, C)}


def bench(C, iters, B=512):
    charset = CHARSET_94[: min(C - 1, 94)] + "".join(chr(0x4E00 + i) for i in range(max(0, C - 1 - 94)))
    cfg = make_config("parseq", charset_train=charset)
    assert cfg.num_classes == C
    eng = Engine(cfg, 0, max_batch=B)
    st = torch.cuda.current_stream().cuda_stream
    eng.load_state_dict(init_state_dict(cfg, 0), st)
    x = synth_images(cfg, B, 1).cuda()
    L = eng.num_steps(None)
    logits = torch.empty((B, L, C), device="cuda")
    ids = torch.empty((B, L), dtype=torch.int32, device="cuda")
    steps = torch.empty((1,), dtype=torch.int32, device="cuda")
    rows = []
    for name, m in masks(charset, B, C).items():
        m = None if m is None else m.cuda()

        def fwd(n):
            eng.forward(x.data_ptr(), n, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, 25, True, 1,
                        class_mask_ptr=None if m is None else m.data_ptr())

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
        rows.append(dict(C=C, mask=name, batch=B, device_img_s=round(B / dev_ms * 1e3), device_ms=round(dev_ms, 3),
                         ar_kernel_ms=round(t["dec_ar"]["ms"], 3), bs1_p50_ms=round(lat[len(lat) // 2], 3)))
    eng.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--classes", default="95,16384")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = []
    c = card()
    for C in (int(v) for v in args.classes.split(",")):
        for r in bench(C, args.iters):
            r["card"] = c
            print(json.dumps(r), flush=True)
            out.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
