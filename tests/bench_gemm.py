"""GEMM microbenchmark (not a test): device time per launch over tile configs, epilogues and K."""
import sys, os, itertools
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check
lib = load_library()
st = torch.cuda.current_stream().cuda_stream

def run(M, N, K, mode, resid_inplace, cg, bn, iters=30, stages=0):
    check(lib, lib.parseq_set_option(None, b"gemm_stages", stages))
    check(lib, lib.parseq_set_option(None, b"cta_group", cg))
    check(lib, lib.parseq_set_option(None, b"block_n", bn))
    A = torch.randn((M, K), device="cuda").bfloat16()
    W = (torch.randn((N, K), device="cuda") * 0.02).bfloat16()
    bias = torch.randn((N,), device="cuda")
    out = torch.zeros((M, N), device="cuda", dtype=torch.float32 if mode == 0 else torch.bfloat16)
    resid = out if resid_inplace else None
    def call():
        check(lib, lib.parseq_gemm_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, N, K, mode, 1.0,
                                        resid.data_ptr() if resid is not None else None, N if resid is not None else 0, 0,
                                        out.data_ptr(), N, st))
    for _ in range(3): call()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): call()
    b.record(); torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1000 / iters
    return us, 2.0 * M * N * K / us / 1e6

M = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
print("shape                mode        cg bn  |    us     TF/s")
cases = [("qkv", 1152, 384, 1, False), ("proj", 384, 384, 0, True), ("fc1", 1536, 384, 2, False), ("fc2", 384, 1536, 0, True)]
for name, N, K, mode, ri in cases:
    for cg, bn in [(1, 128), (1, 192), (1, 256), (2, 256)]:
        if bn == 192 and N % 192: continue
        us, tf = run(M, N, K, mode, ri, cg, bn)
        print(f"{name:5s} N={N:5d} K={K:5d} mode={mode} inplace={int(ri)} cg={cg} bn={bn:3d} | {us:8.1f} {tf:7.1f}")
print("--- K sweep, N=1536 bf16 out (epilogue cost fixed, main loop ~ K)")
for K in (64, 384, 4096):
    for cg, bn in [(1, 128), (1, 256)]:
        us, tf = run(M, 1536, K, 1, False, cg, bn, iters=15)
        print(f"K={K:5d} cg={cg} bn={bn:3d} | {us:8.1f} us {tf:7.1f} TF/s")
print("--- operand-ring depth sweep (gemm_stages cap; full ring: bn256 -> 4, bn192 -> 4, bn128 -> 6)")
for name, N, K, mode, ri in cases:
    for bn, depths in ((256, (2, 3, 4)), (128, (2, 3, 4, 6))):
        for d in depths:
            us, tf = run(M, N, K, mode, ri, 1, bn, 1, stages=d)
            print(f"{name:5s} bn={bn:3d} stages={d} | {us:8.1f} us {tf:7.1f} TF/s")
print("--- cuBLAS reference (torch.matmul bf16, no epilogue)")
for N, K in ((1152, 384), (384, 384), (1536, 384), (384, 1536), (1536, 4096)):
    A = torch.randn((M, K), device="cuda").bfloat16(); W = torch.randn((N, K), device="cuda").bfloat16()
    for _ in range(3): torch.matmul(A, W.t())
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(30): torch.matmul(A, W.t())
    b.record(); torch.cuda.synchronize()
    us = a.elapsed_time(b) * 1000 / 30
    print(f"cublas N={N} K={K}: {us:8.1f} us {2.0*M*N*K/us/1e6:7.1f} TF/s")
