"""Microbenchmark (not a test) of the fused QKV projection + attention kernel against the two kernels it replaces, at the
encoder's shapes (T = 128, head_dim 64): device time per launch of (a) the QKV GEMM, (b) the attention kernel, (c) both
back to back, (d) the fused kernel; the tensor rate, and the HBM bytes the algorithm needs (computed from the shapes) at
that time.

    python tests/bench_qkv_attn.py [B ...]        (default B = 512 images, M = 65 536 rows: PARSeq at bs = 512)"""
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check
lib = load_library()
st = torch.cuda.current_stream().cuda_stream
T = 128


def timeit(fn, iters=50):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000 / iters


def run(B, D):
    M, heads = B * T, D // 64
    xn = torch.randn((M, D), device="cuda").bfloat16()
    W = (torch.randn((3 * D, D), device="cuda") * 0.05).bfloat16()
    bias = torch.randn((3 * D,), device="cuda")
    qkv = torch.empty((M, 3 * D), device="cuda", dtype=torch.bfloat16)
    att = torch.empty((M, D), device="cuda", dtype=torch.bfloat16)
    check(lib, lib.parseq_set_option(None, b"attn_impl", 0))
    qkv_gemm = lambda: check(lib, lib.parseq_gemm_bf16(xn.data_ptr(), D, W.data_ptr(), D, bias.data_ptr(), M, 3 * D, D, 1, 1.0,
                                                       None, 0, 0, qkv.data_ptr(), 3 * D, st))
    attn = lambda: check(lib, lib.parseq_enc_attention(qkv.data_ptr(), B, T, D, heads, att.data_ptr(), st))
    fused = lambda: check(lib, lib.parseq_qkv_attention_bf16(xn.data_ptr(), W.data_ptr(), bias.data_ptr(), B, T, D, heads,
                                                             att.data_ptr(), st))
    f_gemm, f_attn = 2.0 * M * 3 * D * D, 4.0 * B * T * T * D
    b_xn, b_w, b_qkv, b_att = M * D * 2, 3 * D * D * 2, M * 3 * D * 2, M * D * 2
    rows = [("(a) QKV GEMM", qkv_gemm, f_gemm, b_xn + b_w + b_qkv),
            ("(b) attention", attn, f_attn, b_qkv + b_att),
            ("(c) a + b", lambda: (qkv_gemm(), attn()), f_gemm + f_attn, b_xn + b_w + 2 * b_qkv + b_att),
            ("(d) fused", fused, f_gemm + f_attn, b_xn + b_w + b_att)]
    for name, fn, flops, nbytes in rows:
        t = timeit(fn)
        print(f"B={B:4d} D={D} {name:14s} | {t:7.1f} us | {flops / t / 1e6:6.1f} TFLOP/s | HBM {nbytes / 1e6:5.0f} MB "
              f"at {nbytes / t / 1e3:5.0f} GB/s", flush=True)


q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.strip()
print(f"{torch.cuda.get_device_name(0)} | nvidia-smi: {q}", flush=True)
for B in [int(a) for a in sys.argv[1:]] or [512]:
    for D in (384, 192):
        run(B, D)
