"""Raw crops of any size: what the on-device resize costs and what it saves (not a test).

    python tests/bench_crops.py [--steps 20] [--out FILE]

Crop sizes come from a seeded distribution (h in [16, 128], w in [32, 512]), PARSeq-S at 32 x 128, AR + 1 refine pass.
In one run, with the card's name and power limit:
  * device: images/s of model(CUDA crops) (parseq_forward_crops) against model(uint8 stack) (parseq_forward_u8) on
    the same crops resized beforehand, and the resize kernel's time alone (parseq_resize_crops, CUDA events), at
    bs 512 and bs 1;
  * end to end from host memory: images/s of torchvision-PIL T.Resize of each crop on one CPU core + the uint8 host
    path (parseq_forward_host_u8), against model(CPU crops) (packing into pinned memory + parseq_forward_host_crops).
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def ragged(n, seed):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.integers(0, 256, (int(rng.integers(16, 129)), int(rng.integers(32, 513)), 3),
                                         dtype=np.uint8)) for _ in range(n)]


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from PIL import Image
    import torchvision.transforms as T
    from parseq_b200.config import make_config
    from parseq_b200.factory import create_model
    from parseq_b200.system import _crops_c, pack_crops
    from parseq_b200.weights import init_state_dict
    torch.set_num_threads(1)
    cfg = make_config("parseq")
    m = create_model("parseq")
    m.model.load_state_dict(init_state_dict(cfg, 0))
    m = m.eval().to("cuda")
    eng = m.model.engine()
    st = torch.cuda.current_stream().cuda_stream
    resize = T.Resize((32, 128), T.InterpolationMode.BICUBIC)
    res = {"card": card(), "model": "parseq (S), 32x128, AR + 1 refine", "crop_h": [16, 128], "crop_w": [32, 512]}
    with torch.inference_mode():
        for bs in (512, 1):
            crops = ragged(bs, bs)
            dev = [c.cuda() for c in crops]
            pre = m.preprocess(dev)
            data, offsets, sizes = pack_crops(dev)
            cc = _crops_c(data, offsets, sizes, 0)
            out = torch.empty_like(pre)
            steps = args.steps if bs > 1 else 10 * args.steps
            t_crops = timed(lambda: m(dev), steps)
            t_u8 = timed(lambda: m(pre), steps)
            t_resize = timed(lambda: eng.resize_crops(cc, bs, out.data_ptr(), st), steps)
            res[f"bs{bs}"] = {"crops_img_s": bs / t_crops * 1e3, "u8_img_s": bs / t_u8 * 1e3, "crops_ms": t_crops,
                              "u8_ms": t_u8, "resize_kernel_ms": t_resize,
                              "crop_bytes_mb": sum(c.numel() for c in crops) / 1e6}
        bs = 512
        crops = ragged(bs, 7)
        pils = [Image.fromarray(c.numpy()) for c in crops]
        hl = torch.empty((bs, 26, 95), dtype=torch.float32).pin_memory()
        hi = torch.empty((bs, 26), dtype=torch.int32).pin_memory()
        hs = torch.empty((1,), dtype=torch.int32).pin_memory()
        hu = torch.empty((bs, 32, 128, 3), dtype=torch.uint8).pin_memory()

        def pil_path():
            for i, p in enumerate(pils):
                hu[i].copy_(torch.from_numpy(np.asarray(resize(p))))
            eng.forward_u8(hu.data_ptr(), bs, hl.data_ptr(), hi.data_ptr(), hs.data_ptr(), st, None, True, 1, host=True)

        def crops_path():
            m(crops)

        e2e = {}
        for name, fn in (("pil_resize_plus_forward_host_u8", pil_path), ("forward_host_crops", crops_path)):
            fn()
            reps = max(3, args.steps // 4)
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
            e2e[name] = bs * reps / (time.perf_counter() - t0)
        res["e2e_bs512_img_s"] = e2e
        res["e2e_note"] = "PIL resize on one CPU core (torch.set_num_threads(1)); host outputs synchronised per call"
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
