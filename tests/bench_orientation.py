"""Orientation search throughput (parseq_forward_crops_oriented) on PARSeq-S at 95 and 16384 head classes and on
ViTSTR-S: images/s at bs = 512 and p50 ms at bs = 1 for R = 1 (0), R = 2 (0 / 180), R = 4 and the threshold mode at the
t that re-reads about 10 % of the seeded crops (R = 4), alternated in the same process with plain forward(crops) on the
same seeded raw crops, and the device milliseconds per timing category (the orientation kernels included) of one
bs = 512 full R = 4 search.  Head scaled by HEAD_SCALE (below).

    python tests/bench_orientation.py [--out DIR]

Every shape runs once untimed before it is timed; each throughput figure is the best of three windows.  The card's name
and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_score import card  # noqa: E402

REREAD = 0.10
# The seeded weights' head is scaled so that its softmax rows are peaked as a trained model's are: at the seeded scale
# every max probability is near 1 / C and the sequence confidences underflow (all 0 at 16384 classes), so no threshold
# would re-read a chosen fraction.  The work of every call is the same at any scale.
HEAD_SCALE = 12.0


def model(experiment, n_extra):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config_long(experiment, 25, n_extra)
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=25)
    sd = init_state_dict(cfg, 0)
    for k in ("head.weight", "head.bias"):
        sd[k] = sd[k] * HEAD_SCALE
    (m if experiment == "vitstr" else m.model).load_state_dict(sd)
    return cfg, m.eval().to("cuda")


def crops(n, seed):
    """Seeded raw crops of the crop benchmark's distribution (h in [16, 128], w in [32, 512]) on the device."""
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.integers(0, 256, (int(rng.integers(16, 129)), int(rng.integers(32, 513)), 3),
                                         dtype=np.uint8)).cuda() for _ in range(n)]


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
    dev = card()
    print("device:", dev, flush=True)
    rows = []
    for name, experiment, n_extra in (("parseq-s C95", "parseq", 0), ("parseq-s C16384", "parseq", 16289),
                                      ("vitstr-s C95", "vitstr", 0)):
        cfg, m = model(experiment, n_extra)
        c512, c1 = crops(512, 1), crops(1, 2)
        eng = m.model.engine()
        with torch.inference_mode():
            _, _, conf0 = m.read_oriented(c512, (0,))
            # the least t with at least REREAD of the crops below it (random weights give many equal confidences, e.g.
            # products that underflow to 0 at 16384 classes, so the fraction re-read is recorded with t)
            c = torch.sort(conf0.double().cpu()).values
            t = next((float(v) for v in torch.unique(c) if int((c < v).sum()) >= REREAD * len(c)), float(c[-1]))
        runs = {
            "forward(crops)": lambda c: m(c),
            "R=1 (0)": lambda c: m.read_oriented(c, (0,)),
            "R=2 (0, 180)": lambda c: m.read_oriented(c, (0, 180)),
            "R=4": lambda c: m.read_oriented(c, (0, 90, 180, 270)),
            "R=4 threshold": lambda c: m.read_oriented(c, (0, 90, 180, 270), min_confidence=t),
        }
        with torch.inference_mode():
            for key in runs:                               # warm every shape
                runs[key](c512)
                runs[key](c1)
            m.read_oriented(c512, (0, 90, 180, 270), min_confidence=t)
            reread = eng.debug_int("orient_rereads")
            best = {k: float("inf") for k in runs}
            lat = {k: [] for k in runs}
            for _ in range(3):                             # alternate the variants, best of three windows
                for key in runs:
                    best[key] = min(best[key], window(lambda: runs[key](c512), 3))
                    for _ in range(10):
                        lat[key].append(window(lambda: runs[key](c1), 1))
            eng.set_option("timing", 1)
            m.read_oriented(c512, (0, 90, 180, 270))
            torch.cuda.synchronize()
            cats = {c: round(v["ms"], 3) for c, v in eng.get_timing().items() if v["launches"]}
            eng.set_option("timing", 0)
        base = best["forward(crops)"]
        for key in runs:
            r = dict(model=name, variant=key, images_per_s_bs512=round(512 / best[key], 1),
                     time_vs_forward_bs512=round(best[key] / base, 3), p50_ms_bs1=round(1e3 * statistics.median(lat[key]), 3))
            if key == "R=4 threshold":
                r.update(min_confidence=t, reread_crops=reread, reread_fraction=round(reread / 512, 4),
                         confidence_quartiles=[float(x) for x in torch.quantile(conf0.double().cpu(),
                                                                                torch.tensor([0.25, 0.5, 0.75], dtype=torch.float64))])
            rows.append(r)
            print(json.dumps(r), flush=True)
        total = sum(cats.values())
        r = dict(model=name, variant="R=4 device ms per category, bs = 512", categories=cats,
                 orient_share=round(cats.get("orient", 0.0) / total, 4) if total else None)
        rows.append(r)
        print(json.dumps(r), flush=True)
        del m
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_orientation.json"), "w") as f:
            json.dump(dict(device=dev, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
