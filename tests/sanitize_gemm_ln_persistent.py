"""Small driver for compute-sanitizer (not a test):

    compute-sanitizer --tool racecheck|synccheck python tests/sanitize_gemm_ln_persistent.py

The persistent column-split GEMM + LayerNorm kernel (gemm_ln.cuh MODE 2) with several 128-row tiles per cluster, so
that the operand ring, the x buffer and the row-statistics barriers are handed from tile to tile; both K (two- and
four-part row statistics) and a ragged last tile."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check

lib = load_library()
st = torch.cuda.current_stream().cuda_stream
D = 384
clusters = torch.cuda.get_device_properties(0).multi_processor_count // 2
M = 128 * clusters * 3 + 77                      # three to four tiles per cluster
g = torch.Generator(device="cuda").manual_seed(0)
for K in (384, 1536):
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((D, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((D,), device="cuda", generator=g)
    gamma, beta = torch.ones((D,), device="cuda"), torch.zeros((D,), device="cuda")
    x = torch.randn((M, D), device="cuda", generator=g)
    xn = torch.empty((M, D), device="cuda", dtype=torch.bfloat16)
    check(lib, lib.parseq_set_option(None, b"ln_split", 2))
    check(lib, lib.parseq_gemm_ln_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, D, K, x.data_ptr(),
                                       gamma.data_ptr(), beta.data_ptr(), 1e-6, xn.data_ptr(), st))
    torch.cuda.synchronize()
    assert torch.isfinite(x).all() and torch.isfinite(xn.float()).all()
    print("ok: K", K, "M", M, flush=True)
check(lib, lib.parseq_set_option(None, b"ln_split", 0))
print("sanitize_gemm_ln_persistent done")
