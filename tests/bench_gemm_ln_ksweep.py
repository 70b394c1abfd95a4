"""Microbenchmark (not a test): K sweep of the default fused residual-GEMM + LayerNorm kernel at D = 384 (gemm_ln.cuh
MODE 2: persistent CTA pairs on 64-row tiles, ping-pong MMA warpgroups).  The least-squares fit t = a + b * k-blocks
splits a launch into the part that grows with K (the main loops, b per k-block) and the part that does not (a: the
epilogues and the x / xn traffic, as far as they are not hidden under the main loops).

    python tests/bench_gemm_ln_ksweep.py [M]        (default M = 65 536, PARSeq-S at bs = 512)"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check
lib = load_library()
st = torch.cuda.current_stream().cuda_stream
D = 384
TILE_M = 64                                        # rows per tile of MODE 2


def timeit(fn, iters=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000 / iters


def hbm_bytes(M, K):
    """A and W once, x read and written (fp32), xn written (bf16)."""
    return 2 * M * K + 2 * D * K + 2 * 4 * M * D + 2 * M * D


def l2_operand_bytes(M, K):
    """A and W bytes fetched from L2 into shared memory: each CTA of a pair stages the tile's A rows and half of W."""
    tiles = (M + TILE_M - 1) // TILE_M
    return tiles * (2 * TILE_M * K * 2 + D * K * 2)


def run(M, K):
    A = torch.randn((M, K), device="cuda").bfloat16()
    W = (torch.randn((D, K), device="cuda") * 0.02).bfloat16()
    bias = torch.randn((D,), device="cuda"); g = torch.ones((D,), device="cuda"); b = torch.zeros((D,), device="cuda")
    x = torch.randn((M, D), device="cuda"); xn = torch.empty((M, D), device="cuda", dtype=torch.bfloat16)
    t = timeit(lambda: check(lib, lib.parseq_gemm_ln_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, D, K,
                                                          x.data_ptr(), g.data_ptr(), b.data_ptr(), 1e-6, xn.data_ptr(), st)))
    h, l2 = hbm_bytes(M, K), l2_operand_bytes(M, K)
    print(f"M={M:6d} K={K:5d} | {t:7.1f} us | {2.0*M*D*K/t/1e6:6.1f} TF/s | HBM {h/1e6:5.0f} MB at {h/t/1e3:5.0f} GB/s "
          f"| L2->SM operands {l2/1e6:6.0f} MB at {l2/t/1e3:5.0f} GB/s", flush=True)
    return t


print(torch.cuda.get_device_name(0), flush=True)
M = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
Ks = (64, 128, 384, 768, 1536)
kb = np.array([(K + 63) // 64 for K in Ks], dtype=np.float64)
t = np.array([run(M, K) for K in Ks])
slope, icpt = np.polyfit(kb, t, 1)
print(f"K sweep, M={M}: t = {icpt:.1f} us + {slope:.2f} us per k-block (per launch)", flush=True)
clusters = lib.parseq_debug_int(None, b"ln_clusters")   # CTA pairs the launcher used
steps = -(-((M + TILE_M - 1) // TILE_M) // clusters)    # tiles one pair walks
print(f"  {clusters} CTA pairs, {steps} tiles each: {icpt / steps:.2f} us + {slope / steps:.3f} us per k-block per tile",
      flush=True)
