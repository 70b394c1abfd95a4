"""What the cross-attention maps cost (not a test):

    python tests/bench_attn_maps.py [--out FILE]

PARSeq-S (AR + 1 refinement and AR without refinement) at C = 95 and C = 16384 head classes.  In one process, calls
without maps (forward) and with maps (read_with_attention's engine call) alternate, every shape warmed up first:
  * device images/s at bs = 512 (CUDA-graph replay, CUDA events), best of three windows per variant;
  * bs = 1 p50 latency (host clock around a synchronised call), best of three windows;
  * the device ms of one bs = 512 call in timing mode: the maps kernel's category ("attn_maps"), and the whole map pass
    of the AR-only schedule (the timed total with maps minus the total without).
Prints one JSON line per case and writes them, with the card's name and power limit read in the same run, to --out."""
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


def bench(C, refine, iters, B=512):
    charset = CHARSET_94[: min(C - 1, 94)] + "".join(chr(0x4E00 + i) for i in range(max(0, C - 1 - 94)))
    cfg = make_config("parseq", charset_train=charset)
    assert cfg.num_classes == C
    eng = Engine(cfg, 0, max_batch=B)
    st = torch.cuda.current_stream().cuda_stream
    eng.load_state_dict(init_state_dict(cfg, 0), st)
    x = synth_images(cfg, B, 1).cuda()
    L, T = eng.num_steps(None), cfg.num_patches
    logits = torch.empty((B, L, C), device="cuda")
    ids = torch.empty((B, L), dtype=torch.int32, device="cuda")
    steps = torch.empty((1,), dtype=torch.int32, device="cuda")
    maps = torch.empty((B, L, T), device="cuda")

    def fwd(n, with_maps):
        eng.forward(x.data_ptr(), n, logits.data_ptr(), ids.data_ptr(), steps.data_ptr(), st, None, True, refine,
                    attn_maps_ptr=maps.data_ptr() if with_maps else None)

    for n in (B, 1):
        for v in (False, True):
            for _ in range(3):
                fwd(n, v)
    torch.cuda.synchronize()
    best = {False: 0.0, True: 0.0}
    for _ in range(3):
        for v in (False, True):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fwd(B, v)
            b.record()
            torch.cuda.synchronize()
            best[v] = max(best[v], B * iters / (a.elapsed_time(b) * 1e-3))
    lat = {False: float("inf"), True: float("inf")}
    for _ in range(3):
        for v in (False, True):
            w = []
            for _ in range(5 * iters):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fwd(1, v)
                torch.cuda.synchronize()
                w.append((time.perf_counter() - t0) * 1e3)
            w.sort()
            lat[v] = min(lat[v], w[len(w) // 2])
    timed = {}
    for v in (False, True):
        eng.set_option("timing", 1)
        fwd(B, v)
        torch.cuda.synchronize()
        timed[v] = eng.get_timing()
        eng.set_option("timing", 0)
    total = {v: sum(c["ms"] for c in timed[v].values()) for v in (False, True)}
    return {"C": C, "refine_iters": refine, "bs": B,
            "images_per_s": {"forward": round(best[False], 1), "with_maps": round(best[True], 1),
                             "ratio": round(best[True] / best[False], 4)},
            "bs1_p50_ms": {"forward": round(lat[False], 4), "with_maps": round(lat[True], 4)},
            "timed_ms_bs512": {"attn_maps_kernel": round(timed[True]["attn_maps"]["ms"], 4),
                               "attn_maps_launches": timed[True]["attn_maps"]["launches"],
                               "map_pass_total": round(total[True] - total[False], 4),
                               "forward_total": round(total[False], 4)},
            "maps_bytes_bs512": B * L * T * 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    gpu = card()
    rows = []
    for C in (95, 16384):
        for refine in (1, 0):
            r = bench(C, refine, args.iters)
            print(json.dumps(r), flush=True)
            rows.append(r)
    out = {"card": gpu, "note": "timed_ms_bs512: timing mode serialises every launch on one stream; map_pass_total is "
                                "the timed total with maps minus the total without (the maps kernel, and for "
                                "refine_iters 0 the teacher-forced map pass)", "results": rows}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
            f.write("\n")


if __name__ == "__main__":
    main()
