"""Encoder-attention microbenchmark (not a test): device time per launch of the mma.sync kernels (attn_impl 0) and the
wgmma kernel (attn_impl 1) at the token counts of the configurations (T = 128 PARSeq, 129 ViTSTR, 196 patch16-224 without
class token, 240 ViT-B 48x160), ~64 k query rows per launch."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from parseq_b200.build import build
build()
from parseq_b200.engine import load_library, check
lib = load_library()
st = torch.cuda.current_stream().cuda_stream
res = {"device": torch.cuda.get_device_name(0)}
for T, heads in ((128, 6), (129, 6), (196, 6), (240, 12)):
    D = heads * 64
    B = max(1, 65536 // T)
    qkv = (torch.randn((B * T, 3 * D), device="cuda") * 1.5).bfloat16()
    out = torch.empty((B * T, D), dtype=torch.bfloat16, device="cuda")
    for impl in (0, 1):
        check(lib, lib.parseq_set_option(None, b"attn_impl", impl))
        call = lambda: check(lib, lib.parseq_enc_attention(qkv.data_ptr(), B, T, D, heads, out.data_ptr(), st))
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            call()
        b.record()
        torch.cuda.synchronize()
        res[f"T{T}_h{heads}_B{B}_impl{impl}_us"] = round(a.elapsed_time(b) * 1000 / 20, 1)
check(lib, lib.parseq_set_option(None, b"attn_impl", 0))
print(json.dumps(res))
