"""Microbenchmark (not a test) of the fused residual-GEMM + LayerNorm kernel vs the unfused pair: device time per launch."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check
lib = load_library()
st = torch.cuda.current_stream().cuda_stream
D = 384

def timeit(fn, iters=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000 / iters

def run(M, K):
    A = torch.randn((M, K), device="cuda").bfloat16()
    W = (torch.randn((D, K), device="cuda") * 0.02).bfloat16()
    bias = torch.randn((D,), device="cuda"); g = torch.ones((D,), device="cuda"); b = torch.zeros((D,), device="cuda")
    x = torch.randn((M, D), device="cuda"); xn = torch.empty((M, D), device="cuda", dtype=torch.bfloat16)
    fused = lambda: check(lib, lib.parseq_gemm_ln_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, D, K, x.data_ptr(),
                                                       g.data_ptr(), b.data_ptr(), 1e-6, xn.data_ptr(), st))
    gemm = lambda: check(lib, lib.parseq_gemm_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, D, K, 0, 1.0, x.data_ptr(), D, 0,
                                                   x.data_ptr(), D, st))
    ln = lambda: check(lib, lib.parseq_layernorm_bf16(x.data_ptr(), g.data_ptr(), b.data_ptr(), 1e-6, M, D, xn.data_ptr(), None, st))
    tf, tg, tl = timeit(fused), timeit(gemm), timeit(ln)
    print(f"M={M:6d} K={K:5d} | fused {tf:7.1f} us ({2.0*M*D*K/tf/1e6:6.1f} TF/s) | gemm {tg:7.1f} + ln {tl:5.1f} = {tg+tl:7.1f} us", flush=True)

for cg, pdl, split in ((1, 0, 1), (2, 0, 1), (1, 0, 2)):
    check(lib, lib.parseq_set_option(None, b"ln_cta_group", cg))
    check(lib, lib.parseq_set_option(None, b"pair_pdl", pdl))
    check(lib, lib.parseq_set_option(None, b"ln_split", split))
    print(f"--- fused kernel: ln_cta_group={cg} pair_pdl={pdl} ln_split={split} (2 = column-split pair)", flush=True)
    for M in (65536, 132 * 128 * 4):
        for K in (384, 1536, 4096):
            run(M, K)
