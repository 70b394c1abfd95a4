"""Candidate scoring throughput (parseq_score) on PARSeq-S and ViTSTR-S: images/s and candidates/s, the device time of
the encoder, decoder, LayerNorm + other and scoring-tail categories, and the tail's achieved TFLOP/s.

    python tests/bench_score.py [--out DIR]

Workloads: bs = 512 with a shared seeded lexicon of 3-12-character words, K in {1, 10, 100}, at 95 and 16384 head
classes; bs = 1 with K = 10; ViTSTR-S at bs = 512, K in {10, 100}.  Every workload runs once untimed before any is
timed; each figure is the best of three timed windows.  At K = 10 (95 classes) the scorer is alternated, in the
same process, with the workaround a user has without it - every image repeated K times through `forward` with the
candidates as teacher-forced ids and refine_iters = 0, then log_softmax of the [N K, 26, C] logits and a gather - and
with plain `forward` (AR + 1 refine) on the same images.  The card's name and power limit are read in the same run and printed with every number."""
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

ENC = ("enc_gemm", "enc_attn", "enc_gemm_ln")
DEC = ("dec_gemm", "dec_attn")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def model(n_extra, experiment="parseq"):
    from make_golden_long import charset, make_config_long
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    cfg = make_config_long(experiment, 25, n_extra)
    m = create_model(experiment, charset_train=charset(n_extra), max_label_length=25)
    (m if experiment == "vitstr" else m.model).load_state_dict(init_state_dict(cfg, 0))
    return cfg, m.eval().to("cuda")


def lexicon(k, seed=0):
    from make_golden_long import charset
    cs = charset(0)
    r = np.random.default_rng(seed)
    return ["".join(cs[i] for i in r.integers(0, 94, r.integers(3, 13))) for _ in range(k)]


def timed(fn, iters, warmup=2, repeats=1):
    """Seconds per call: the best of `repeats` windows of `iters` calls, after `warmup` untimed calls."""
    for _ in range(warmup):
        fn()
    best = float("inf")
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
        best = min(best, (time.perf_counter() - t) / iters)
    return best


def split(m, fn):
    eng = m.model.engine()
    eng.set_option("timing", 0)
    eng.set_option("timing", 1)
    fn()
    torch.cuda.synchronize()
    t = eng.get_timing()
    eng.set_option("timing", 0)
    # LayerNorm and "other" (gathers, im2col) serve both the encoder and the decoder: reported on their own
    tail = t["score_tail"]
    return dict(encoder_ms=sum(t[k]["ms"] for k in ENC), decoder_ms=sum(t[k]["ms"] for k in DEC),
                ln_other_ms=t["layernorm"]["ms"] + t["other"]["ms"], tail_ms=tail["ms"],
                tail_tflops=tail["flops"] / (tail["ms"] * 1e-3) / 1e12 if tail["ms"] > 0 else None)


def workaround(m, x, lex):
    """Repeat every image K times, force the candidates through the AR loop (refine_iters = 0), log_softmax + gather."""
    tok = m.tokenizer
    K, N = len(lex), x.shape[0]
    L = 26
    ids = torch.full((K, L), tok.pad_id, dtype=torch.int32)
    tgt = torch.zeros((K, L), dtype=torch.long)
    for k, w in enumerate(lex):
        r = [tok.bos_id] + tok._tok2ids(w) + [tok.eos_id]
        ids[k, :min(len(r), L)] = torch.tensor(r[:L], dtype=torch.int32)
        tgt[k, :len(w) + 1] = torch.tensor(tok._tok2ids(w) + [0])
    valid = (torch.arange(L)[None, :] <= torch.tensor([len(w) for w in lex])[:, None])
    ids, tgt, valid = ids.repeat(N, 1).cuda(), tgt.repeat(N, 1).cuda(), valid.repeat(N, 1).cuda()
    xr = x.repeat_interleave(K, 0)

    def run():
        logits = m.model.forward(tok, xr, 25, forced_ids=ids)
        lp = torch.log_softmax(logits, -1).gather(2, tgt[..., None])[..., 0]
        return (lp * valid).sum(-1).view(N, K)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    from parseq_b200.weights import synth_images
    gpu = card()
    rows = []
    runs = [("parseq", 0), ("parseq", 16289), ("vitstr", 0)]
    for exp, n_extra in runs:
        cfg, m = model(n_extra, exp)
        C = cfg.num_classes
        x512 = synth_images(cfg, 512, 1).cuda()
        work = [(512, 1), (512, 10), (512, 100), (1, 10)] if exp == "parseq" else [(512, 10), (512, 100)]
        with torch.inference_mode():
            for N, K in work:                                                        # every workload once, untimed
                m.score(x512[:N], lexicon(K))
            for N, K in work:
                x = x512[:N]
                lex = lexicon(K)
                fn = lambda: m.score(x, lex)                                         # noqa: E731
                sec = timed(fn, args.iters if N * K < 20000 else max(3, args.iters // 3), repeats=3)
                r = dict(gpu=gpu, model=exp, classes=C, batch=N, K=K, ms=sec * 1e3, images_per_s=N / sec,
                         candidates_per_s=N * K / sec, **split(m, fn))
                rows.append(r)
                print(json.dumps(r), flush=True)
            if exp == "parseq" and n_extra == 0:
                lex = lexicon(10)
                base = workaround(m, x512, lex)
                m.model.refine_iters = 0
                s_ref = m.score(x512, lex)
                diff = (base() - s_ref).abs().max().item()
                m.model.refine_iters = 1
                t_s, t_w, t_f = [], [], []
                for _ in range(3):                                                   # alternated in one process
                    t_s.append(timed(lambda: m.score(x512, lex), args.iters))
                    m.model.refine_iters = 0
                    t_w.append(timed(base, max(2, args.iters // 3), warmup=1))
                    m.model.refine_iters = 1
                    t_f.append(timed(lambda: m(x512), args.iters))
                r = dict(gpu=gpu, classes=C, batch=512, K=10, score_ms=min(t_s) * 1e3, workaround_ms=min(t_w) * 1e3,
                         forward_ms=min(t_f) * 1e3, speedup_vs_workaround=min(t_w) / min(t_s),
                         score_over_forward=min(t_s) / min(t_f), max_abs_diff_vs_workaround=diff,
                         spread_score=(max(t_s) - min(t_s)) / min(t_s), spread_workaround=(max(t_w) - min(t_w)) / min(t_w))
                rows.append(r)
                print(json.dumps(r), flush=True)
        del m
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_score.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
