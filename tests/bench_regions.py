"""Cost of reading text regions of full frames (crop_regions, parseq_warp_regions) on PARSeq-S.

Workload: 512 seeded regions, 20-120 px tall and 60-800 px wide, turned by up to 45 degrees with mild perspective (each
corner moved by up to 5 % of the height), from four 1920 x 1080 frames and one 3840 x 2160 frame (blocky seeded pixels),
the regions spread over the five frames in turn.  Reported, each the best of three windows, the variants alternated in
one process after every shape has run once untimed:
  * the warp kernel alone: ms by CUDA events around parseq_warp_regions (the table upload included), and its byte
    floor: the crops' bytes written once plus the same number read (a region reads about one source pixel per output
    pixel), over the data sheet's 3.35 TB/s;
  * crop_regions as a Python call (argument checks, coefficients, frame packing, the kernel);
  * model(model.crop_regions(frames, quads)) against model(crops) on the same regions already cut (separate CUDA
    tensors);
  * the CPU route: PIL's Image.transform(PERSPECTIVE, BICUBIC) of every region on one core, then model(PIL crops).
The card's name and power limit are read in the same run and stored with the numbers.

    python tests/bench_regions.py [--out tests/results/bench_regions_h100.json]"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import make_golden_regions as mg  # noqa: E402
from bench_score import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
FRAMES = [(1080, 1920)] * 4 + [(2160, 3840)]


def workload(n=512, seed=0):
    rng = np.random.default_rng(seed)
    frames = [mg.make_frame(H, W, 200 + k, 4) for k, (H, W) in enumerate(FRAMES)]
    quads, index = [], []
    while len(quads) < n:
        f = len(quads) % len(FRAMES)
        H, W = FRAMES[f]
        th = rng.uniform(-math.pi / 4, math.pi / 4)
        h, w = rng.uniform(20, 120), rng.uniform(60, 800)
        q = mg.rect(rng.uniform(0, W), rng.uniform(0, H), w, h, math.cos(th), math.sin(th))
        q = [(x + rng.uniform(-0.05, 0.05) * h, y + rng.uniform(-0.05, 0.05) * h) for x, y in q]
        if mg.convex(q):
            quads.append(q)
            index.append(f)
    return frames, np.array(quads, dtype=np.float64), np.array(index, dtype=np.int64)


def window(fn, iters):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "results", "bench_regions_h100.json"))
    args = ap.parse_args()
    from PIL import Image
    from parseq_b200.config import make_config
    from parseq_b200.engine import RegionsC
    from parseq_b200.factory import create_model
    from parseq_b200.weights import init_state_dict
    torch.set_num_threads(1)
    dev_name = card()
    print("device:", dev_name, flush=True)
    cfg = make_config("parseq")
    m = create_model("parseq")
    m.model.load_state_dict(init_state_dict(cfg, 0))
    m = m.eval().to("cuda")
    frames_np, quads, index = workload()
    frames = [torch.from_numpy(f).cuda() for f in frames_np]
    pil_frames = [Image.fromarray(f) for f in frames_np]
    with torch.inference_mode():
        rc = m.crop_regions(frames, quads, frame_index=index)
        precut = [c.clone() for c in rc]
        out_bytes = int(rc.data.numel())
        # the kernel alone: the same call parseq_warp_regions gets from crop_regions, on prepared arguments
        eng = m.model.engine()
        fdata = torch.cat([f.reshape(-1) for f in frames])
        fsz = torch.tensor([f.shape[:2] for f in frames_np], dtype=torch.int32)
        fnb = 3 * fsz[:, 0].long() * fsz[:, 1].long()
        foff = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(fnb, 0)[:-1]])
        fi32 = torch.from_numpy(index.astype(np.int32))
        rc_c = RegionsC(fdata.data_ptr(), fdata.numel(), foff.data_ptr(), fsz.data_ptr(), len(frames), fi32.data_ptr(),
                        rc.sizes.data_ptr(), rc.coeffs.data_ptr())
        out = torch.empty(out_bytes, dtype=torch.uint8, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def kernel_ms(iters=50):
            ev0.record()
            for _ in range(iters):
                eng.warp_regions(rc_c, len(quads), out.data_ptr(), out_bytes, stream)
            ev1.record()
            ev1.synchronize()
            return ev0.elapsed_time(ev1) / iters

        def pil_route():
            crops = []
            for q, f in zip(quads, index):
                h, w = q_sizes[len(crops)]
                crops.append(pil_frames[f].transform((w, h), Image.Transform.PERSPECTIVE,
                                                     tuple(rc.coeffs[len(crops)].tolist()), Image.Resampling.BICUBIC))
            return m(crops)

        q_sizes = [tuple(s) for s in rc.sizes.tolist()]
        runs = {
            "crop_regions": lambda: m.crop_regions(frames, quads, frame_index=index),
            "model(crop_regions)": lambda: m(m.crop_regions(frames, quads, frame_index=index)),
            "model(precut crops)": lambda: m(precut),
        }
        kernel_ms(5)
        assert torch.equal(out, rc.data), "the timed kernel call must make crop_regions' bytes"
        for fn in runs.values():
            fn()
        pil_route()
        best = {k: float("inf") for k in list(runs) + ["warp kernel", "CPU route (PIL + model(PIL crops))"]}
        for _ in range(3):
            best["warp kernel"] = min(best["warp kernel"], kernel_ms() / 1e3)
            for k, fn in runs.items():
                best[k] = min(best[k], window(fn, 5))
            best["CPU route (PIL + model(PIL crops))"] = min(best["CPU route (PIL + model(PIL crops))"],
                                                             window(pil_route, 1))
    floor_s = 2 * out_bytes / HBM_BYTES_PER_S
    pixels = out_bytes // 3
    rows = []
    for k, t in best.items():
        r = dict(variant=k, ms=round(1e3 * t, 4), regions_per_s=round(len(quads) / t, 1))
        if k == "warp kernel":
            r.update(out_bytes=out_bytes, output_pixels=pixels, byte_floor_ms=round(1e3 * floor_s, 4),
                     share_of_byte_floor=round(floor_s / t, 4))
        rows.append(r)
        print(json.dumps(r), flush=True)
    res = dict(device=dev_name, model="parseq-s (seeded weights)", regions=len(quads),
               frames=[list(f) for f in FRAMES], method="best of 3 windows, alternated; warp kernel by CUDA events over "
               "50 calls, the rest by host clock around 5 calls ending in a synchronise (CPU route: 1 call)", rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
