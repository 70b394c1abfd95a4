"""GPU: the fused QKV projection + attention kernel (qkv_attn.cuh) computes the bits of the two-kernel pair it replaces,
the QKV GEMM (bf16 epilogue) followed by the mma.sync attention kernel, and keeps a non-finite image to itself."""
import os
import shutil
import subprocess

import pytest
import torch

pytestmark = pytest.mark.gpu

T = 128
UNSUPPORTED = -2


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _inputs(B, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xn = torch.randn((B * T, D), device="cuda", generator=g).bfloat16()
    W = (torch.randn((3 * D, D), device="cuda", generator=g) * 0.08).bfloat16()
    bias = torch.randn((3 * D,), device="cuda", generator=g) * 0.5
    return xn, W, bias


def _pair(lib, xn, W, bias, B, D):
    from parseq_b200.engine import check
    check(lib, lib.parseq_set_option(None, b"attn_impl", 0))
    qkv = torch.empty((B * T, 3 * D), dtype=torch.bfloat16, device="cuda")
    check(lib, lib.parseq_gemm_bf16(xn.data_ptr(), D, W.data_ptr(), D, bias.data_ptr(), B * T, 3 * D, D, 1, 1.0, None, 0, 0,
                                    qkv.data_ptr(), 3 * D, _stream()))
    out = torch.empty((B * T, D), dtype=torch.bfloat16, device="cuda")
    check(lib, lib.parseq_enc_attention(qkv.data_ptr(), B, T, D, D // 64, out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return out


def _fused(lib, xn, W, bias, B, D):
    from parseq_b200.engine import check
    out = torch.full((B * T, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    check(lib, lib.parseq_qkv_attention_bf16(xn.data_ptr(), W.data_ptr(), bias.data_ptr(), B, T, D, D // 64, out.data_ptr(),
                                             _stream()))
    torch.cuda.synchronize()
    return out


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("D", [192, 384])
@pytest.mark.parametrize("B", [1, 2, 7, 133, 512])
def test_fused_qkv_attention_is_byte_equal_to_the_pair(lib, B, D):
    """One item, fewer items than CTAs, several items per CTA and a ragged last round of the persistent grid."""
    xn, W, bias = _inputs(B, D, B * 1000 + D)
    ref = _pair(lib, xn, W, bias, B, D)
    out = _fused(lib, xn, W, bias, B, D)
    assert bool(torch.isfinite(ref.float()).all())
    diff = (_bits(out) != _bits(ref)).any(dim=1).nonzero().flatten()
    assert diff.numel() == 0, f"{diff.numel()} rows differ, first {diff[:8].tolist()}"


@pytest.mark.parametrize("D", [192, 384])
def test_fused_qkv_attention_nonfinite_image_stays_in_its_rows(lib, D):
    """NaN / inf in one image's xn rows: every other image's rows keep the bits of the clean run and of the pair."""
    B, bad = 7, 3
    xn, W, bias = _inputs(B, D, 77 + D)
    clean = _fused(lib, xn, W, bias, B, D)
    dirty = xn.clone()
    dirty[bad * T + 5, 17] = float("nan")
    dirty[bad * T + 90, 3] = float("inf")
    dirty[bad * T + 91, D - 1] = float("-inf")
    out = _fused(lib, dirty, W, bias, B, D)
    ref = _pair(lib, dirty, W, bias, B, D)
    keep = torch.ones(B * T, dtype=torch.bool, device="cuda")
    keep[bad * T:(bad + 1) * T] = False
    assert torch.equal(_bits(out)[keep], _bits(clean)[keep])
    assert torch.equal(_bits(out)[keep], _bits(ref)[keep])
    assert not bool(torch.isfinite(out[~keep].float()).all())


def test_fused_qkv_attention_rejects_other_geometries(lib):
    xn, W, bias = _inputs(2, 384, 5)
    out = torch.empty((2 * 129, 384), dtype=torch.bfloat16, device="cuda")
    for t, d, heads in ((129, 384, 6), (240, 384, 6), (128, 768, 12), (128, 384, 3), (128, 256, 4)):
        rc = lib.parseq_qkv_attention_bf16(xn.data_ptr(), W.data_ptr(), bias.data_ptr(), 2, t, d, heads, out.data_ptr(),
                                           _stream())
        assert rc == UNSUPPORTED, (t, d, heads)


def test_fused_qkv_attention_sass():
    """wgmma (HGMMA) for the QKV projection, TMA loads (UTMALDG) into the operand ring, mma.sync (HMMA) for the attention."""
    from parseq_b200.build import LIB_PATH, build
    build()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", LIB_PATH], capture_output=True, text=True).stdout
    fn = [b for b in sass.split("Function : ")[1:] if "enc_qkv_attn_kernel" in b.split("\n", 1)[0]]
    assert len(fn) == 2                       # D in {192, 384}
    for body in fn:
        for mnemonic in ("HGMMA", "UTMALDG", "HMMA"):
            assert mnemonic in body, mnemonic
