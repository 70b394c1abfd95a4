"""Beam search throughput (parseq_beam_search) on PARSeq-S at 95 and 16384 head classes and on ViTSTR-S: images/s at
bs = 512 and p50 ms at bs = 1 for beam widths 1, 4, 8 and 16, alternated in the same process with greedy `forward`
(refine_iters = 0; the default AR path and the chain of separate kernels, ar_kernel = 0) on the same seeded images,
and the device milliseconds per timing category (beam_select included) of one bs = 512 call.

    python tests/bench_beam.py [--out DIR]

Every shape runs once untimed before it is timed; each throughput figure is the best of three windows.  The card's name
and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_score import card  # noqa: E402


def model(experiment, n_extra):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config_long(experiment, 25, n_extra)
    kw = {} if experiment == "vitstr" else {"refine_iters": 0}
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=25, **kw)
    (m if experiment == "vitstr" else m.model).load_state_dict(init_state_dict(cfg, 0))
    return cfg, m.eval().to("cuda")


def window(fn, iters):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from parseq_b200.weights import synth_images
    dev = card()
    print("device:", dev, flush=True)
    rows = []
    for name, experiment, n_extra in (("parseq-s C95", "parseq", 0), ("parseq-s C16384", "parseq", 16289),
                                      ("vitstr-s C95", "vitstr", 0)):
        cfg, m = model(experiment, n_extra)
        x512 = synth_images(cfg, 512, 1).cuda()
        x1 = x512[:1].contiguous()
        eng = m.model.engine()
        runs = {}
        for K in (1, 4, 8, 16):
            runs[f"beam K={K}"] = (lambda x, K=K: m.model.beam_search(x, K), None)
        if experiment == "vitstr":
            runs["greedy forward"] = (lambda x: m.model.forward_tokens(x, None), None)
        else:
            runs["greedy forward"] = (lambda x: m.model.forward(m.tokenizer, x, 25), 2)
            runs["greedy forward chain"] = (lambda x: m.model.forward(m.tokenizer, x, 25), 0)

        def run(key, x):
            fn, ark = runs[key]
            if ark is not None:
                m.model.set_engine_option("ar_kernel", ark)
            return fn(x)
        with torch.inference_mode():
            for key in runs:                               # warm every shape
                run(key, x512)
                run(key, x1)
            best = {k: float("inf") for k in runs}
            lat = {k: [] for k in runs}
            for _ in range(3):                             # alternate the variants, best of three windows
                for key in runs:
                    best[key] = min(best[key], window(lambda: run(key, x512), 2))
                    for _ in range(10):
                        lat[key].append(window(lambda: run(key, x1), 1))
            cats = {}
            for K in (1, 16):
                eng.set_option("timing", 0)
                eng.set_option("timing", 1)
                m.model.beam_search(x512, K)
                torch.cuda.synchronize()
                cats[K] = {c: round(v["ms"], 3) for c, v in eng.get_timing().items() if v["launches"]}
                eng.set_option("timing", 0)
        for key in runs:
            r = dict(model=name, variant=key, images_per_s_bs512=round(512 / best[key], 1),
                     p50_ms_bs1=round(1e3 * statistics.median(lat[key]), 3))
            rows.append(r)
            print(json.dumps(r), flush=True)
        for K, c in cats.items():
            r = dict(model=name, variant=f"beam K={K} device ms per category, bs = 512", categories=c)
            rows.append(r)
            print(json.dumps(r), flush=True)
        del m
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_beam.json"), "w") as f:
            json.dump(dict(device=dev, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
