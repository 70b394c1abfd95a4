"""Microbenchmark (not a test) of the fused residual-GEMM + LayerNorm kernel at the encoder's shapes (D = 384, attn.proj
K = 384, mlp.fc2 K = 1536): device time per launch, the rate against the HBM bytes the algorithm needs, and the operand
bytes each kernel moves from L2 to the SMs, computed from the shapes.

    python tests/bench_gemm_ln_roofline.py [M ...]        (default M = 65 536, PARSeq-S at bs = 512)"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check
lib = load_library()
st = torch.cuda.current_stream().cuda_stream
D = 384


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


def l2_operand_bytes(M, K, ln_split):
    """A and W bytes fetched from L2 into shared memory (a multicast box counts once)."""
    if ln_split == 1:                              # full-row kernel: 64-row CTAs, each stages all of W
        tiles = (M + 63) // 64
        return tiles * (64 * K * 2 + D * K * 2)
    tiles = (M + 127) // 128                       # column-split pairs: A multicast, each CTA stages half of W
    return tiles * (128 * K * 2 + D * K * 2)


def run(M, K, ln_split):
    A = torch.randn((M, K), device="cuda").bfloat16()
    W = (torch.randn((D, K), device="cuda") * 0.02).bfloat16()
    bias = torch.randn((D,), device="cuda"); g = torch.ones((D,), device="cuda"); b = torch.zeros((D,), device="cuda")
    x = torch.randn((M, D), device="cuda"); xn = torch.empty((M, D), device="cuda", dtype=torch.bfloat16)
    check(lib, lib.parseq_set_option(None, b"ln_split", ln_split))
    t = timeit(lambda: check(lib, lib.parseq_gemm_ln_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, D, K,
                                                          x.data_ptr(), g.data_ptr(), b.data_ptr(), 1e-6, xn.data_ptr(), st)))
    check(lib, lib.parseq_set_option(None, b"ln_split", 0))
    h, l2 = hbm_bytes(M, K), l2_operand_bytes(M, K, ln_split)
    print(f"M={M:6d} K={K:5d} ln_split={ln_split} | {t:7.1f} us | {2.0*M*D*K/t/1e6:6.1f} TF/s | HBM {h/1e6:5.0f} MB "
          f"at {h/t/1e3:5.0f} GB/s | L2->SM operands {l2/1e6:6.0f} MB at {l2/t/1e3:5.0f} GB/s", flush=True)


print(torch.cuda.get_device_name(0), flush=True)
for M in [int(a) for a in sys.argv[1:]] or [65536]:
    for K in (384, 1536):
        for ln_split in (0, 1):                    # 0: the default (column-split pairs at D = 384), 1: full-row kernel
            run(M, K, ln_split)
