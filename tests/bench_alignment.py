"""The cost of character maps for given text: score, beam search and locate(text=) with maps against the same calls
without, on PARSeq-S at 95 and 16384 head classes, bs = 512.

    python tests/bench_alignment.py [--out DIR] [--iters N]

Workloads: `score` with a shared seeded lexicon of 3-12-character words at K = 1, 10 and 100 candidates per image,
beam search at K = 4 and 16, and locate(text=) with one word per image, set against `score` of the same words and
against `locate` of the greedy reading, whose per-image centre / box code it shares.  Each call with maps is alternated
with the same call without, in one process, after one untimed call of each; each figure is the best of `iters` calls.  In
timing mode (every launch serialised on one stream) the grouped maps kernel's device time is read from the "attn_maps"
category and set against its byte floor: the K it stages (T x D bf16 per CTA, one CTA per image and 32 map rows), the q
rows it reads and the maps it writes, over 3.35 TB/s.  The card's name and power limit are read in the same run and
recorded with every number."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_BYTES_PER_S = 3.35e12
AMAP_ROWS = 32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def model(n_extra):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config_long("parseq", 25, n_extra)
    m = create_model("parseq", charset_train=charset(n_extra), max_label_length=25)
    m.model.load_state_dict(init_state_dict(cfg, 0))
    return cfg, m.eval().to("cuda")


def lexicon(k, seed=0):
    from make_golden_long import charset
    cs = charset(0)
    r = np.random.default_rng(seed)
    return ["".join(cs[i] for i in r.integers(0, 94, r.integers(3, 13))) for _ in range(k)]


def alternate(fns, iters):
    """Best seconds per call of each fn, the fns alternated call by call after one untimed call each."""
    for f in fns:
        f()
    best = [float("inf")] * len(fns)
    for _ in range(iters):
        for i, f in enumerate(fns):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            best[i] = min(best[i], time.perf_counter() - t0)
    return best


def timed_categories(m, fn):
    eng = m.model.engine()
    eng.set_option("timing", 1)
    fn()
    torch.cuda.synchronize()
    t = eng.get_timing()
    eng.set_option("timing", 0)
    return t


def score_floor_bytes(cfg, B, K, words):
    """Bytes the grouped maps kernel must move for B images of the same K words: each CTA stages the image's K (T x D
    bf16), the computed rows' q (fp32 D) are read once, the maps (fp32 L x T per candidate) written once."""
    L, T, D = cfg.max_label_length + 1, cfg.num_patches, cfg.embed_dim
    ctas = B * -(-K * L // AMAP_ROWS)
    rows = B * sum(len(w) + 1 for w in words)
    return ctas * T * D * 2 + rows * D * 4 + B * K * L * T * 4


def run(n_extra, B, iters):
    cfg, m = model(n_extra)
    from parseq_b200.weights import synth_images
    x = synth_images(cfg, B, 0).cuda()
    out = {"C": cfg.num_classes, "bs": B, "score": {}, "beam": {}}
    with torch.inference_mode():
        for K in (1, 10, 100):
            words = lexicon(K, K)
            f0 = lambda: m.score(x, words)                                       # noqa: E731
            f1 = lambda: m.score(x, words, return_attention=True)                # noqa: E731
            t0, t1 = alternate([f0, f1], iters)
            cat = timed_categories(m, f1)["attn_maps"]
            floor = score_floor_bytes(cfg, B, K, words)
            out["score"][f"K{K}"] = {
                "ms": {"without_maps": round(t0 * 1e3, 3), "with_maps": round(t1 * 1e3, 3),
                       "ratio": round(t1 / t0, 4)},
                "maps_kernel": {"ms": round(cat["ms"], 4), "launches": cat["launches"], "floor_bytes": floor,
                                "floor_ms": round(floor / HBM_BYTES_PER_S * 1e3, 4),
                                "share_of_floor": round(floor / HBM_BYTES_PER_S * 1e3 / cat["ms"], 4) if cat["ms"] else None}}
        for K in (4, 16):
            f0 = lambda: m.beam_search(x, K)                                     # noqa: E731
            f1 = lambda: m.beam_search(x, K, return_attention=True)              # noqa: E731
            t0, t1 = alternate([f0, f1], iters)
            cat = timed_categories(m, f1)["attn_maps"]
            out["beam"][f"K{K}"] = {"ms": {"without_maps": round(t0 * 1e3, 3), "with_maps": round(t1 * 1e3, 3),
                                           "ratio": round(t1 / t0, 4)},
                                    "maps_kernel_ms": round(cat["ms"], 4), "maps_launches": cat["launches"]}
        texts = lexicon(B, 7)
        f0 = lambda: m.score(x, [[t] for t in texts])                            # noqa: E731
        f1 = lambda: m.locate(x, text=texts)                                     # noqa: E731
        f2 = lambda: m.locate(x)                                                 # noqa: E731
        t0, t1, t2 = alternate([f0, f1, f2], iters)
        out["locate_text"] = {"ms": {"score_without_maps": round(t0 * 1e3, 3), "locate_text": round(t1 * 1e3, 3),
                                     "locate_greedy": round(t2 * 1e3, 3), "ratio_to_score": round(t1 / t0, 4)}}
    m.model.engine().close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--bs", type=int, default=512)
    a = ap.parse_args()
    gpu = card()
    res = {"card": gpu, "note": "ms: best host-clocked call, with and without maps alternated in one process; "
                                "maps_kernel: device ms of the attn_maps category in timing mode (launches serialised)",
           "workloads": [run(n, a.bs, a.iters) for n in (0, 16289)]}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_alignment_h100.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
