"""Cost of reading curved text regions of full frames (crop_regions with polygons, parseq_warp_polygons) on PARSeq-S.

Workload: 512 seeded curved words, arcs of k = 7 and k = 16 points per edge in turn (14 and 32 points), 20-120 px tall
and 60-800 px long along the arc, bent by 10-90 degrees either way, from four 1920 x 1080 frames and one 3840 x 2160
frame (blocky seeded pixels), the regions spread over the five frames in turn.  Reported, each the best of three
windows, the variants alternated in one process after every shape has run once untimed:
  * region_tps_kernel alone, by CUDA events around parseq_warp_polygons (coefficient solve and table upload included),
    against region_warp_kernel (parseq_warp_regions) on quads of exactly the same crop sizes and frames;
  * crop_regions as a Python call (checks, engine order, coefficients, frame packing, the kernel);
  * model(model.crop_regions(frames, polygons)) against model(crops) on the same crops already cut;
  * the CPU route on one core, timed on the first 64 regions and scaled to 512: per region the fp64 TPS grid of
    GridGenerator's numpy builders (as restated in tests/tps_warp_oracle.py, since the reference tree is not installed
    where this runs), torch's grid_sample (bicubic, zeros outside) and PIL's resize to the model's input size.
The card's name and power limit are read in the same run and stored with the numbers.

    python tests/bench_curved_regions.py [--out tests/results/bench_curved_regions_h100.json]"""
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

import make_golden_curved as mgc  # noqa: E402
import make_golden_regions as mg  # noqa: E402
from bench_score import card  # noqa: E402

FRAMES = [(1080, 1920)] * 4 + [(2160, 3840)]
CPU_ROUTE_REGIONS = 64                      # the CPU route is timed on the first 64 regions and scaled to all of them


def workload(n=512, seed=0):
    from parseq_b200.regions import check_polygon
    rng = np.random.default_rng(seed)
    frames = [mg.make_frame(H, W, 300 + k, 4) for k, (H, W) in enumerate(FRAMES)]
    polys, index = [], []
    while len(polys) < n:
        f = len(polys) % len(FRAMES)
        H, W = FRAMES[f]
        k = 7 if len(polys) % 2 == 0 else 16
        length, half = rng.uniform(60, 800), rng.uniform(10, 60)
        bend = math.radians(rng.uniform(10, 90)) * rng.choice([-1, 1])
        r = length / abs(bend)
        a0 = rng.uniform(-110, -70) if bend > 0 else rng.uniform(70, 110)
        cx, cy = rng.uniform(0, W), rng.uniform(0, H)
        span = math.degrees(bend)
        p = mgc.band(mgc.arc(cx, cy + (r if bend > 0 else -r), r, a0 - span / 2, a0 + span / 2), k, half)
        try:
            check_polygon(p)
        except ValueError:
            continue
        polys.append(np.array(p))
        index.append(f)
    return frames, polys, np.array(index, dtype=np.int64)


def window(fn, iters):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "results", "bench_curved_regions_h100.json"))
    args = ap.parse_args()
    import torch.nn.functional as F
    from PIL import Image
    from parseq_b200.config import make_config
    from parseq_b200.engine import PolygonsC, RegionsC
    from parseq_b200.factory import create_model
    from parseq_b200.regions import engine_points, quad_coeffs
    from parseq_b200.weights import init_state_dict
    from tps_warp_oracle import tps_map
    torch.set_num_threads(1)
    dev_name = card()
    print("device:", dev_name, flush=True)
    cfg = make_config("parseq")
    m = create_model("parseq")
    m.model.load_state_dict(init_state_dict(cfg, 0))
    m = m.eval().to("cuda")
    frames_np, polys, index = workload()
    frames = [torch.from_numpy(f).cuda() for f in frames_np]
    with torch.inference_mode():
        rc = m.crop_regions(frames, polys, frame_index=index)
        precut = [c.clone() for c in rc]
        out_bytes = int(rc.data.numel())
        sizes = [tuple(s) for s in rc.sizes.tolist()]
        eng = m.model.engine()
        fdata = torch.cat([f.reshape(-1) for f in frames])
        fsz = torch.tensor([f.shape[:2] for f in frames_np], dtype=torch.int32)
        fnb = 3 * fsz[:, 0].long() * fsz[:, 1].long()
        foff = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(fnb, 0)[:-1]])
        fi32 = torch.from_numpy(index.astype(np.int32))
        pts = [engine_points(p.tolist()) for p in polys]
        npt = torch.tensor([len(p) for p in pts], dtype=torch.int32)
        flat = torch.tensor([xy for p in pts for xy in p], dtype=torch.float64)
        pc = PolygonsC(fdata.data_ptr(), fdata.numel(), foff.data_ptr(), fsz.data_ptr(), len(frames), fi32.data_ptr(),
                       rc.sizes.data_ptr(), npt.data_ptr(), flat.data_ptr())
        # quads of the same crop sizes: each polygon's chord rectangle, turned like it, with the polygon's (h, w)
        qcf = []
        for p, (h, w) in zip(pts, sizes):
            k = len(p) // 2
            (x0, y0), (x1, y1) = p[0], p[k - 1]
            th = math.atan2(y1 - y0, x1 - x0)
            q = mg.rect((x0 + x1) / 2, (y0 + y1) / 2, w, h, math.cos(th), math.sin(th))
            qcf.append(quad_coeffs(q, h, w))
        qcf = torch.tensor(qcf, dtype=torch.float64)
        rq = RegionsC(fdata.data_ptr(), fdata.numel(), foff.data_ptr(), fsz.data_ptr(), len(frames), fi32.data_ptr(),
                      rc.sizes.data_ptr(), qcf.data_ptr())
        out = torch.empty(out_bytes, dtype=torch.uint8, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def events_ms(call, iters=50):
            ev0.record()
            for _ in range(iters):
                call()
            ev1.record()
            ev1.synchronize()
            return ev0.elapsed_time(ev1) / iters

        def tps_call():
            eng.warp_polygons(pc, len(pts), out.data_ptr(), out_bytes, stream)

        def quad_call():
            eng.warp_regions(rq, len(pts), out.data_ptr(), out_bytes, stream)

        img_w, img_h = cfg.img_size[1], cfg.img_size[0]
        frames_t = [torch.from_numpy(f).permute(2, 0, 1)[None].double() for f in frames_np]

        def cpu_route():
            res = []
            for p, f, (h, w) in list(zip(pts, index, sizes))[:CPU_ROUTE_REGIONS]:
                from parseq_b200.engine import tps_coeffs
                X, Y = tps_map(tps_coeffs(p), h, w)
                H, W = frames_np[f].shape[:2]
                grid = torch.from_numpy(np.stack([2.0 * X / W - 1.0, 2.0 * Y / H - 1.0], -1))[None]
                c = F.grid_sample(frames_t[f], grid, mode="bicubic", padding_mode="zeros", align_corners=False)
                c = c[0].permute(1, 2, 0).clamp(0, 255).to(torch.uint8).numpy()
                res.append(Image.fromarray(c).resize((img_w, img_h), Image.Resampling.BICUBIC))
            return res

        runs = {
            "crop_regions": lambda: m.crop_regions(frames, polys, frame_index=index),
            "model(crop_regions)": lambda: m(m.crop_regions(frames, polys, frame_index=index)),
            "model(precut crops)": lambda: m(precut),
        }
        events_ms(tps_call, 3)
        assert torch.equal(out, rc.data), "the timed kernel call must make crop_regions' bytes"
        events_ms(quad_call, 3)
        for fn in runs.values():
            fn()
        cpu_route()
        names = ["region_tps_kernel", "region_warp_kernel (same sizes)"] + list(runs) + \
            ["CPU route (TPS grid + grid_sample + PIL resize, 1 core)"]
        best = {k: float("inf") for k in names}
        for _ in range(3):
            best["region_tps_kernel"] = min(best["region_tps_kernel"], events_ms(tps_call) / 1e3)
            best["region_warp_kernel (same sizes)"] = min(best["region_warp_kernel (same sizes)"], events_ms(quad_call) / 1e3)
            for k, fn in runs.items():
                best[k] = min(best[k], window(fn, 5))
            best[names[-1]] = min(best[names[-1]], window(cpu_route, 1) * len(pts) / CPU_ROUTE_REGIONS)
    pixels = out_bytes // 3
    rows = []
    for k, t in best.items():
        r = dict(variant=k, ms=round(1e3 * t, 4), regions_per_s=round(len(pts) / t, 1))
        if "kernel" in k:
            r.update(output_pixels=pixels, ns_per_pixel=round(1e9 * t / pixels, 4))
        rows.append(r)
        print(json.dumps(r), flush=True)
    res = dict(device=dev_name, model="parseq-s (seeded weights)", regions=len(pts),
               points_per_region=sorted(set(npt.tolist())), output_pixels=pixels,
               frames=[list(f) for f in FRAMES], method="best of 3 windows, alternated; kernels by CUDA events over "
               "50 calls (host coefficient solve and table upload included), the rest by host clock around 5 calls "
               "ending in a synchronise (CPU route: 1 call over the first 64 regions, scaled to 512)", rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
