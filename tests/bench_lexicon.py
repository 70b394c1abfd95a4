"""Lexicon-constrained beam search throughput (parseq_beam_search_lexicon): images/s at bs = 512 and p50 ms at bs = 1.

  - PARSeq-S at 95 classes: per-image lexicons of 50 words and shared lexicons of 1 000 and 50 000 seeded words at beam
    widths 1, 4 and 16, alternated in the same process with plain beam search at the same widths and with exhaustive
    lexicon decoding (every word scored, `score`) for the 50- and 1 000-word lexicons;
  - PARSeq-S at 16384 classes with a 20 000-word lexicon of CJK-style 2-4 character words, and ViTSTR-S with the
    1 000-word lexicon, against plain beam search.
Also the host trie build time and device bytes of each lexicon, and the top-1 agreement of the beam pick with the
exhaustive pick on the 1 000-word lexicon (bs = 512, with the seeded head bias of the beam goldens), with the mean score
gap between the two picks.

    python tests/bench_lexicon.py [--out DIR]

Every shape runs once untimed before it is timed; each throughput figure is the best of three windows.  The card's name
and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import random
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_beam import model, window  # noqa: E402
from bench_score import card  # noqa: E402


def words(cs, n, seed, lo, hi):
    rng = random.Random(seed)
    out = set()
    while len(out) < n:
        out.add("".join(rng.choice(cs) for _ in range(rng.randint(lo, hi))))
    return sorted(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from make_golden_long import charset
    from parseq_b200.system import pack_candidates
    from parseq_b200.weights import synth_images
    dev = card()
    print("device:", dev, flush=True)
    rows = []
    for name, experiment, n_extra in (("parseq-s C95", "parseq", 0), ("parseq-s C16384", "parseq", 16289),
                                      ("vitstr-s C95", "vitstr", 0)):
        cfg, m = model(experiment, n_extra)
        cs = charset(n_extra)
        x512 = synth_images(cfg, 512, 1).cuda()
        x1 = x512[:1].contiguous()
        if n_extra:
            lexicons = {"shared 20k": words(cs[94:], 20000, 3, 2, 4)}
        elif experiment == "parseq":
            lexicons = {"per-image 50": [words(cs, 50, 100 + b, 3, 10) for b in range(512)],
                        "shared 1k": words(cs, 1000, 4, 3, 10), "shared 50k": words(cs, 50000, 5, 3, 12)}
        else:
            lexicons = {"shared 1k": words(cs, 1000, 4, 3, 10)}
        compiled = {}
        for key, ws in lexicons.items():
            t = time.perf_counter()
            lex = m.compile_lexicon(ws)
            build_ms = 1e3 * (time.perf_counter() - t)
            compiled[key] = lex
            r = dict(model=name, lexicon=key, trie_build_ms=round(build_ms, 1), nodes=lex.num_nodes, edges=lex.num_edges,
                     device_bytes=lex.nbytes)
            rows.append(r)
            print(json.dumps(r), flush=True)
        runs = {}
        Ks = (1, 4, 16)
        for K in Ks:
            runs[f"beam K={K}"] = lambda x, K=K: m.model.beam_search(x, K)
            for key, lex in compiled.items():
                def fn(x, K=K, lex=lex):
                    roots = lex.roots_for(x.shape[0]) if lex.roots is not None and x.shape[0] > 1 else (
                        lex.roots[:1] if lex.roots is not None else None)
                    return m.model.beam_search(x, K, lexicon=lex, roots=roots)
                runs[f"lexicon {key} K={K}"] = fn
        if experiment == "parseq" and not n_extra:
            for key in ("per-image 50", "shared 1k"):
                packed = {}
                for B in (512, 1):
                    ws = lexicons[key]
                    cands = ws[:B] if isinstance(ws[0], list) else ws
                    packed[B] = pack_candidates(m.tokenizer, cands, B, 25, cfg.num_classes)

                def ex(x, packed=packed):
                    t, n, per = packed[x.shape[0]]
                    return m.model.score(x, t, n, per)
                runs[f"exhaustive score {key}"] = ex
        with torch.inference_mode():
            for key in runs:                               # warm every shape
                runs[key](x512)
                runs[key](x1)
            best = {k: float("inf") for k in runs}
            lat = {k: [] for k in runs}
            for _ in range(3):                             # alternate the variants, best of three windows
                for key in runs:
                    best[key] = min(best[key], window(lambda: runs[key](x512), 2))
                    for _ in range(10):
                        lat[key].append(window(lambda: runs[key](x1), 1))
            agree = {}
            if "shared 1k" in lexicons and experiment == "parseq":
                # The timed weights' rows are nearly flat (hundreds of words within fp32 noise of the best), so the
                # agreement is taken with the goldens' seeded head bias, which spreads the classes as a trained head
                # does.  Two lexicons: the 1 000 random words, where the best word is often one the model reads poorly
                # (its first characters rank low and leave the beam), and the same words plus each image's
                # unconstrained top-1 beam reading, as when the lexicon holds the word the model sees.
                from make_golden_beam import golden_state_dict
                m.model.load_state_dict(golden_state_dict(cfg, 0, 2.0))
                reads, _ = m.beam_search(x512, 16)
                seen = sorted(set(lexicons["shared 1k"]) | {h[0] for h in reads if h and len(h[0]) <= 25})
                for key, ws in (("random 1k", lexicons["shared 1k"]), ("1k + readings", seen)):
                    ex_labels, ex_s = m.lexicon_decode(x512, ws)
                    lex = m.compile_lexicon(ws)
                    for K in Ks:
                        bl, bs = m.lexicon_decode(x512, lex, beam_width=K)
                        agree[(key, K)] = (sum(a == b for a, b in zip(bl, ex_labels)) / 512,
                                           round(float((ex_s - bs).mean()), 4))
        for key in runs:
            r = dict(model=name, variant=key, images_per_s_bs512=round(512 / best[key], 1),
                     p50_ms_bs1=round(1e3 * statistics.median(lat[key]), 3))
            rows.append(r)
            print(json.dumps(r), flush=True)
        for (key, K), (v, gap) in agree.items():
            r = dict(model=name, variant=f"top-1 agreement with exhaustive, lexicon {key}, K={K}, bs = 512", agreement=v,
                     mean_score_gap=gap)
            rows.append(r)
            print(json.dumps(r), flush=True)
        eng = m.model.engine()
        r = dict(model=name, variant="beam_bytes after the lexicon runs", beam_bytes=eng.debug_int("beam_bytes"))
        rows.append(r)
        print(json.dumps(r), flush=True)
        del m
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_lexicon_h100.json"), "w") as f:
            json.dump(dict(device=dev, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
