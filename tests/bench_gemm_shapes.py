"""GEMM microbenchmark (not a test): device time per launch over the encoder's shapes, epilogues and K.

Run it with PARSEQ_B200_LIB pointing at another build of the library to compare two builds on one card.

Prints the card and its power limit first (a rate means nothing without them), then, at M = 65 536 rows (PARSeq-S,
bs = 512, T = 128), TFLOP/s and achieved GB/s for the encoder's GEMM shapes in the epilogue modes the engine runs them
in, a K sweep that separates the fixed per-tile epilogue cost from the main loop, an operand-ring depth sweep and
cuBLAS (torch.matmul, no epilogue) on the same shapes.  GB/s counts the algorithmic bytes: A + W + the output (+ the
fp32 residual read for the in-place residual modes).

    python tests/bench_gemm_shapes.py [M]
"""
import sys, os, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check
lib = load_library()
st = torch.cuda.current_stream().cuda_stream

MODE_NAME = {0: "f32", 1: "bf16", 2: "gelu"}


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        smi = q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi failed"
    except (OSError, IndexError, subprocess.TimeoutExpired):
        smi = "nvidia-smi not available"
    return f"{name} | name, power limit, max SM clock: {smi}"


def timed(call, min_ms=150.0):
    """us per call: warm up, size the window to about min_ms of device time, CUDA events around it."""
    for _ in range(3): call()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); call(); b.record(); torch.cuda.synchronize()
    iters = max(5, min(400, int(min_ms / max(a.elapsed_time(b), 1e-3))))
    a.record()
    for _ in range(iters): call()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000 / iters


def run(M, N, K, mode, resid_inplace, stages=0, min_ms=150.0):
    check(lib, lib.parseq_set_option(None, b"gemm_stages", stages))
    A = torch.randn((M, K), device="cuda").bfloat16()
    W = (torch.randn((N, K), device="cuda") * 0.02).bfloat16()
    bias = torch.randn((N,), device="cuda")
    out = torch.zeros((M, N), device="cuda", dtype=torch.float32 if mode == 0 else torch.bfloat16)
    resid = out if resid_inplace else None
    def call():
        check(lib, lib.parseq_gemm_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, N, K, mode, 1.0,
                                        resid.data_ptr() if resid is not None else None, N if resid is not None else 0, 0,
                                        out.data_ptr(), N, st))
    us = timed(call, min_ms)
    nbytes = M * K * 2 + N * K * 2 + M * N * out.element_size() * (2 if resid_inplace else 1)
    return us, 2.0 * M * N * K / us / 1e6, nbytes / us / 1e3


M = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
print("card:", card())
print(f"M = {M}")
print("--- encoder shapes")
print("shape                              mode |       us    TF/s    GB/s")
# (name, N, K, epilogue mode, in-place fp32 residual): QKV -> bf16, attn.proj -> fp32 + x, fc1 -> GELU bf16,
# fc2 -> fp32 + x, patch embedding (K = 3 x 4 x 8) -> fp32 + pos_embed (here: the plain residual)
cases = [("qkv", 1152, 384, 1, False), ("proj", 384, 384, 0, True), ("fc1", 1536, 384, 2, False),
         ("fc2", 384, 1536, 0, True), ("patch", 384, 96, 0, True)]
for name, N, K, mode, ri in cases:
    us, tf, gbs = run(M, N, K, mode, ri)
    print(f"{name:5s} N={N:5d} K={K:5d} inplace={int(ri)}     {MODE_NAME[mode]:4s} | {us:8.1f} {tf:7.1f} {gbs:7.0f}")
print("--- K sweep, N=1536 bf16 out (epilogue cost fixed per tile, main loop ~ K)")
for K in (64, 384, 4096):
    us, tf, gbs = run(M, 1536, K, 1, False)
    print(f"K={K:5d} | {us:8.1f} us {tf:7.1f} TF/s {gbs:7.0f} GB/s")
print("--- operand-ring depth sweep (gemm_stages cap)")
for name, N, K, mode, ri in cases[:4]:
    for d in (2, 3, 4, 0):
        us, tf, gbs = run(M, N, K, mode, ri, stages=d, min_ms=50.0)
        print(f"{name:5s} stages={d if d else 'full'} | {us:8.1f} us {tf:7.1f} TF/s")
check(lib, lib.parseq_set_option(None, b"gemm_stages", 0))
print("--- cuBLAS reference (torch.matmul bf16 -> bf16, no bias / epilogue)")
for N, K in ((1152, 384), (384, 384), (1536, 384), (384, 1536), (384, 96), (1536, 64), (1536, 4096)):
    A = torch.randn((M, K), device="cuda").bfloat16(); W = torch.randn((N, K), device="cuda").bfloat16()
    us = timed(lambda: torch.matmul(A, W.t()))
    gbs = (M * K * 2 + N * K * 2 + M * N * 2) / us / 1e3
    print(f"cublas N={N:5d} K={K:5d}: {us:8.1f} us {2.0*M*N*K/us/1e6:7.1f} TF/s {gbs:7.0f} GB/s")
