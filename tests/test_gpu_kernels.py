"""Building-block parity on the GPU: every kernel called through the C ABI (include/parseq_b200.h)
and compared with a plain fp32 PyTorch evaluation of the same op on the same bf16-rounded inputs."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gemm(lib, A, W, bias, mode, alpha=1.0, resid=None, resid_mod=0, out=None, ldo=None):
    from parseq_b200.engine import check
    M, K = A.shape
    N = W.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32 if mode == 0 else torch.bfloat16, device=A.device)
    ldo = out.stride(0) if ldo is None else ldo
    check(lib, lib.parseq_gemm_bf16(A.data_ptr(), A.stride(0), W.data_ptr(), W.stride(0),
                                    bias.data_ptr() if bias is not None else None, M, N, K, mode, alpha,
                                    resid.data_ptr() if resid is not None else None,
                                    resid.stride(0) if resid is not None else 0, resid_mod, out.data_ptr(), ldo,
                                    _stream()))
    torch.cuda.synchronize()
    return out


SHAPES = [
    # M, N, K
    (128, 128, 64), (128, 128, 384), (256, 384, 384), (1024, 1152, 384), (512, 1536, 384), (384, 384, 1536),
    (1, 384, 384), (26, 384, 384), (52, 1536, 384), (300, 95, 384), (2522, 768, 384), (640, 384, 96),
    (130, 576, 192), (129, 192, 768), (20000, 384, 384), (4096, 768, 384),
    (700, 1536, 384), (8192, 1152, 384), (1000, 384, 1536), (130, 95, 384),
]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_f32_bias(lib, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((N, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((N,), device="cuda", generator=g)
    ref = A.float() @ W.float().t() + bias
    out = _gemm(lib, A, W, bias, 0)
    err = (out - ref).abs().max().item()
    assert err <= 2e-4 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("N,K,mode", [(1152, 384, 1), (384, 384, 0), (1536, 384, 2), (384, 1536, 0)])
def test_gemm_deterministic_many_tiles_per_cta(lib, N, K, mode):
    """Persistent kernel, ~15-40 tiles per CTA, asynchronous TMA-store epilogue: repeated launches must be bit-identical
    (catches staging-buffer reuse races) and equal to the reference."""
    g = torch.Generator(device="cuda").manual_seed(N + K)
    M = 32768
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((N, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((N,), device="cuda", generator=g)
    outs = []
    for _ in range(4):
        if mode == 0:
            x = torch.ones((M, N), device="cuda")
            outs.append(_gemm(lib, A, W, bias, 0, resid=x, out=x).clone())
        else:
            outs.append(_gemm(lib, A, W, bias, mode).clone())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    acc = A.float() @ W.float().t() + bias
    ref = acc + 1.0 if mode == 0 else (torch.nn.functional.gelu(acc) if mode == 2 else acc)
    err = (outs[0].float() - ref).abs().max().item()
    assert err <= (2e-4 if mode == 0 else 2 ** -7) * ref.abs().max().item(), err


def test_gemm_residual_inplace_and_broadcast(lib):
    g = torch.Generator(device="cuda").manual_seed(5)
    M, N, K = 640, 384, 384
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((N, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((N,), device="cuda", generator=g)
    x = torch.randn((M, N), device="cuda", generator=g)
    ref = x + (A.float() @ W.float().t() + bias)
    out = _gemm(lib, A, W, bias, 0, resid=x, out=x)            # in place (x += ...)
    assert (out - ref).abs().max().item() <= 2e-4 * ref.abs().max().item()
    table = torch.randn((128, N), device="cuda", generator=g)  # residual row = row % 128 (pos_embed pattern)
    ref2 = (A.float() @ W.float().t() + bias) * 0.25 + table.repeat(M // 128, 1)
    out2 = _gemm(lib, A, W, bias, 0, alpha=0.25, resid=table, resid_mod=128)
    assert (out2 - ref2).abs().max().item() <= 2e-4 * ref2.abs().max().item()


def test_gemm_bf16_and_gelu(lib):
    g = torch.Generator(device="cuda").manual_seed(9)
    M, N, K = 384, 1536, 384
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((N, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((N,), device="cuda", generator=g)
    acc = A.float() @ W.float().t() + bias
    out = _gemm(lib, A, W, bias, 1).float()
    assert (out - acc).abs().max().item() <= 2 ** -7 * acc.abs().max().item()      # one bf16 ulp
    assert (out == acc.bfloat16().float()).float().mean().item() > 0.995            # rounding flips only
    ref = torch.nn.functional.gelu(acc)
    out = _gemm(lib, A, W, bias, 2).float()
    assert (out - ref).abs().max().item() <= 2 ** -7 * ref.abs().max().item()
    assert (out == ref.bfloat16().float()).float().mean().item() > 0.99


def test_gemm_head_layout(lib):
    """N=95 (odd row pitch -> scalar store path), strided rows (one AR step of [B, L, C] logits)."""
    g = torch.Generator(device="cuda").manual_seed(11)
    B, L, C, K = 37, 26, 95, 384
    A = torch.randn((B, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((C, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((C,), device="cuda", generator=g)
    logits = torch.zeros((B, L, C), device="cuda")
    step = 7
    _gemm(lib, A, W, bias, 0, out=logits[:, step], ldo=L * C)
    ref = A.float() @ W.float().t() + bias
    assert (logits[:, step] - ref).abs().max().item() <= 2e-4 * ref.abs().max().item()
    logits[:, step] = 0
    assert logits.abs().max().item() == 0.0       # nothing written outside the step's rows


def _gemm_ln(lib, A, W, bias, x, gamma, beta, eps):
    from parseq_b200.engine import check
    M, K = A.shape
    D = W.shape[0]
    xn = torch.empty((M, D), dtype=torch.bfloat16, device=A.device)
    check(lib, lib.parseq_gemm_ln_bf16(A.data_ptr(), A.stride(0), W.data_ptr(), W.stride(0), bias.data_ptr(), M, D, K,
                                       x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps, xn.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return xn


@pytest.fixture(params=[1, 2], ids=["full-row-cta", "column-split-pair"])
def ln_split(request, lib):
    """gemm_ln.cuh: one CTA owns full rows / the columns of a tile split over a CTA pair (D = 384 only)."""
    from parseq_b200.engine import check
    check(lib, lib.parseq_set_option(None, b"ln_split", request.param))
    yield request.param
    check(lib, lib.parseq_set_option(None, b"ln_split", 0))


@pytest.mark.parametrize("M,D,K", [(128, 384, 384), (300, 384, 384), (4096, 384, 1536), (77, 384, 1536),
                                   (148 * 128 * 2 + 77, 384, 384), (65536, 384, 1536), (513, 192, 192), (2000, 192, 768)])
def test_gemm_ln_fused(lib, ln_split, M, D, K):
    """x += A W^T + b (fp32 in place) and xn = bf16(LayerNorm(x)) in one kernel (gemm_ln.cuh) vs the same two ops in torch;
    ragged M, several tiles per CTA, both K of the encoder (attn.proj, mlp.fc2)."""
    g = torch.Generator(device="cuda").manual_seed(M + D + K)
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((D, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((D,), device="cuda", generator=g)
    gamma = 1.0 + 0.1 * torch.randn((D,), device="cuda", generator=g)
    beta = 0.05 * torch.randn((D,), device="cuda", generator=g)
    x0 = torch.randn((M, D), device="cuda", generator=g) + 0.3 * torch.randn((M, 1), device="cuda", generator=g)
    x = x0.clone()
    xn = _gemm_ln(lib, A, W, bias, x, gamma, beta, 1e-6)
    ref_x = x0 + (A.float() @ W.float().t() + bias)
    errx = (x - ref_x).abs().max().item()
    assert errx <= 2e-4 * max(1.0, ref_x.abs().max().item()), ("x", errx)
    # the LayerNorm half is checked on the kernel's own x (isolates it from the GEMM summation order)
    ref_n = torch.nn.functional.layer_norm(x, (D,), gamma, beta, 1e-6)
    errn = (xn.float() - ref_n).abs()
    assert (errn <= 2.0 ** -8 * ref_n.abs() + 1e-5).all(), ("xn", errn.max().item())       # one bf16 rounding
    same = (xn == ref_n.bfloat16()).float().mean().item()
    assert same > 0.995, same                                                               # ties at rounding boundaries only
    x2 = x0.clone()
    xn2 = _gemm_ln(lib, A, W, bias, x2, gamma, beta, 1e-6)
    assert torch.equal(x, x2) and torch.equal(xn, xn2)                                       # deterministic


@pytest.mark.parametrize("M,D,K", [(128, 384, 384), (129, 384, 1536), (300, 384, 384), (148 * 128 + 77, 384, 1536), (65536, 384, 1536),
                                   (513, 192, 192), (2000, 192, 768)])
def test_gemm_ln_cta_pair_equals_single_cta(lib, M, D, K):
    """The fused GEMM + LayerNorm kernel on CTA pairs (each CTA loads half of the W tile and multicasts it into both) returns
    the bits of the single-CTA kernel: same k order per output element, same epilogue.  Ragged M: the last pair tile has
    an empty second CTA / a partial first one."""
    from parseq_b200.engine import check
    g = torch.Generator(device="cuda").manual_seed(M + D + K + 1)
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((D, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((D,), device="cuda", generator=g)
    gamma = 1.0 + 0.1 * torch.randn((D,), device="cuda", generator=g)
    beta = 0.05 * torch.randn((D,), device="cuda", generator=g)
    x0 = torch.randn((M, D), device="cuda", generator=g)
    out = {}
    try:
        check(lib, lib.parseq_set_option(None, b"ln_split", 1))         # the full-row kernel, not the column-split one
        for cg in (1, 2):
            check(lib, lib.parseq_set_option(None, b"ln_cta_group", cg))
            x = x0.clone()
            out[cg] = (x, _gemm_ln(lib, A, W, bias, x, gamma, beta, 1e-6))
    finally:
        check(lib, lib.parseq_set_option(None, b"ln_cta_group", 0))
        check(lib, lib.parseq_set_option(None, b"ln_split", 0))
    assert torch.equal(out[1][0], out[2][0])
    assert torch.equal(out[1][1], out[2][1])
    ref_x = x0 + (A.float() @ W.float().t() + bias)
    assert (out[2][0] - ref_x).abs().max().item() <= 2e-4 * max(1.0, ref_x.abs().max().item())


def _mlp_ln(lib, xn, W1, b1, W2, b2, x, gamma, beta, eps, out=None):
    from parseq_b200.engine import check
    M, D = xn.shape
    xo = torch.empty((M, D), dtype=torch.bfloat16, device=xn.device) if out is None else out
    check(lib, lib.parseq_mlp_ln_bf16(xn.data_ptr(), W1.data_ptr(), b1.data_ptr(), W2.data_ptr(), b2.data_ptr(), M, D, x.data_ptr(),
                                      gamma.data_ptr(), beta.data_ptr(), eps, xo.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return xo


@pytest.fixture(params=[1, 2], ids=["single-cta", "cta-pair"])
def mlp_cta_group(request, lib):
    from parseq_b200.engine import check
    check(lib, lib.parseq_set_option(None, b"mlp_cta_group", request.param))
    yield request.param
    check(lib, lib.parseq_set_option(None, b"mlp_cta_group", 0))


@pytest.mark.parametrize("M,D", [(128, 384), (129, 384), (256, 384), (300, 384), (77, 384), (148 * 128 * 2 + 77, 384), (65536, 384), (513, 192),
                                 (20000, 192)])
def test_mlp_ln_fused_equals_two_kernels(lib, mlp_cta_group, M, D):
    """fc1 + GELU + fc2 + residual + LayerNorm in one kernel (mlp_ln.cuh; the hidden activation stays on the SM) returns
    the bits of the two-kernel path (GEMM with the GELU epilogue, then the fused residual-GEMM + LayerNorm): same k order
    per output element, same rounding points (bf16 hidden, fp32 x, bf16 xn).  Also in place (xn_out aliases xn), and against
    an fp32 torch restatement of the block's MLP (modules: timm Mlp + Block residual + LayerNorm)."""
    H = 4 * D
    g = torch.Generator(device="cuda").manual_seed(M + D)
    xn = torch.randn((M, D), device="cuda", generator=g).bfloat16()
    W1 = (torch.randn((H, D), device="cuda", generator=g) * 0.06).bfloat16()
    b1 = 0.2 * torch.randn((H,), device="cuda", generator=g)
    W2 = (torch.randn((D, H), device="cuda", generator=g) * 0.04).bfloat16()
    b2 = 0.2 * torch.randn((D,), device="cuda", generator=g)
    gamma = 1.0 + 0.1 * torch.randn((D,), device="cuda", generator=g)
    beta = 0.05 * torch.randn((D,), device="cuda", generator=g)
    x0 = torch.randn((M, D), device="cuda", generator=g)
    # two kernels
    hid = torch.empty((M, H), dtype=torch.bfloat16, device="cuda")
    _gemm(lib, xn, W1, b1, 2, out=hid)
    xa = x0.clone()
    from parseq_b200.engine import check
    check(lib, lib.parseq_set_option(None, b"ln_split", 1))     # the full-row GEMM + LayerNorm kernel, whose epilogue mlp_ln.cuh shares
    try:
        xna = _gemm_ln(lib, hid, W2, b2, xa, gamma, beta, 1e-6)
    finally:
        check(lib, lib.parseq_set_option(None, b"ln_split", 0))
    # one kernel
    xb = x0.clone()
    xnb = _mlp_ln(lib, xn, W1, b1, W2, b2, xb, gamma, beta, 1e-6)
    assert torch.equal(xa, xb), (xa - xb).abs().max().item()
    assert torch.equal(xna, xnb)
    # in place: the normalised rows overwrite the kernel's own input
    xc = x0.clone()
    buf = xn.clone()
    _mlp_ln(lib, buf, W1, b1, W2, b2, xc, gamma, beta, 1e-6, out=buf)
    assert torch.equal(xc, xb) and torch.equal(buf, xnb)
    # fp32 restatement (hidden rounded to bf16 like every implementation that stores it)
    h32 = torch.nn.functional.gelu(xn.float() @ W1.float().t() + b1).bfloat16().float()
    ref_x = x0 + (h32 @ W2.float().t() + b2)
    assert (xb - ref_x).abs().max().item() <= 2e-3 * max(1.0, ref_x.abs().max().item())
    ref_n = torch.nn.functional.layer_norm(xb, (D,), gamma, beta, 1e-6)
    assert ((xnb.float() - ref_n).abs() <= 2.0 ** -8 * ref_n.abs() + 1e-5).all()


def test_gemm_ln_fused_matches_unfused_pair(lib, ln_split):
    """Same rounding points as the TMA reduce-add GEMM epilogue followed by layernorm_kernel: x bit-identical."""
    from parseq_b200.engine import check
    M, D, K = 3000, 384, 1536
    g = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((D, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((D,), device="cuda", generator=g)
    gamma = 1.0 + 0.1 * torch.randn((D,), device="cuda", generator=g)
    beta = 0.05 * torch.randn((D,), device="cuda", generator=g)
    x0 = torch.randn((M, D), device="cuda", generator=g)
    xa = x0.clone()
    xna = _gemm_ln(lib, A, W, bias, xa, gamma, beta, 1e-6)
    xb = x0.clone()
    _gemm(lib, A, W, bias, 0, resid=xb, out=xb)
    xnb = torch.empty((M, D), dtype=torch.bfloat16, device="cuda")
    check(lib, lib.parseq_layernorm_bf16(xb.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-6, M, D, xnb.data_ptr(), None,
                                         _stream()))
    torch.cuda.synchronize()
    assert torch.equal(xa, xb)
    assert (xna == xnb).float().mean().item() > 0.999
    assert (xna.float() - xnb.float()).abs().max().item() <= 2.0 ** -7 * xnb.float().abs().max().item()


@pytest.mark.parametrize("D,eps", [(192, 1e-6), (384, 1e-6), (384, 1e-5), (768, 1e-5)])
def test_layernorm(lib, D, eps):
    from parseq_b200.engine import check
    g = torch.Generator(device="cuda").manual_seed(D)
    M = 1000
    x = torch.randn((M, D), device="cuda", generator=g) * 3 + 0.5
    gamma = torch.randn((D,), device="cuda", generator=g)
    beta = torch.randn((D,), device="cuda", generator=g)
    y = torch.empty((M, D), dtype=torch.bfloat16, device="cuda")
    y32 = torch.empty((M, D), dtype=torch.float32, device="cuda")
    check(lib, lib.parseq_layernorm_bf16(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), eps, M, D, y.data_ptr(),
                                         y32.data_ptr(), _stream()))
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x, (D,), gamma, beta, eps)
    assert (y32 - ref).abs().max().item() <= 2e-5
    assert (y.float() == y32.bfloat16().float()).all()


@pytest.fixture
def attn_impl(request, lib):
    """Encoder attention: 1 = the wgmma kernel (attn_wgmma.cuh), 0 = the mma.sync kernels (kernels.cuh, the default), which
    later tests in the same process get back."""
    from parseq_b200.engine import check
    check(lib, lib.parseq_set_option(None, b"attn_impl", request.param))
    yield request.param
    check(lib, lib.parseq_set_option(None, b"attn_impl", 0))


ATTN_IMPLS = pytest.mark.parametrize("attn_impl", [1, 0], ids=["wgmma", "mma_sync"], indirect=True)


@ATTN_IMPLS
@pytest.mark.parametrize("B,heads", [(1, 6), (5, 6), (3, 3), (2, 12), (300, 6)])
def test_enc_attention(lib, B, heads, attn_impl):
    from parseq_b200.engine import check
    T, d = 128, 64
    D = heads * d
    g = torch.Generator(device="cuda").manual_seed(B * 10 + heads)
    qkv = (torch.randn((B * T, 3 * D), device="cuda", generator=g) * 1.5).bfloat16()
    out = torch.empty((B * T, D), dtype=torch.bfloat16, device="cuda")
    check(lib, lib.parseq_enc_attention(qkv.data_ptr(), B, T, D, heads, out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    q, k, v = qkv.float().reshape(B, T, 3, heads, d).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * (d ** -0.5)
    e = torch.exp(s - s.max(-1, keepdim=True).values)
    o = (e.bfloat16().float() @ v) / e.sum(-1, keepdim=True)
    ref = o.permute(0, 2, 1, 3).reshape(B * T, D)
    err = (out.float() - ref).abs().max().item()
    assert err <= 2 ** -7 * ref.abs().max().item() + 1e-3, err


@ATTN_IMPLS
@pytest.mark.parametrize("B,heads,T", [(2, 6, 196), (3, 12, 240), (1, 3, 130), (2, 6, 64), (40, 6, 129), (2, 6, 256), (3, 3, 49)])
def test_enc_attention_any_token_count(lib, B, heads, T, attn_impl):
    """Geometries that do not fill one 128-row tile per image: the wgmma kernel with 128 or 256 keys per tile and one
    CTA per (image, head, 128-query tile), and the masked two-pass mma.sync kernel."""
    from parseq_b200.engine import check
    d = 64
    D = heads * d
    g = torch.Generator(device="cuda").manual_seed(B * 10 + heads + T)
    qkv = (torch.randn((B * T, 3 * D), device="cuda", generator=g) * 1.5).bfloat16()
    out = torch.zeros((B * T, D), dtype=torch.bfloat16, device="cuda")
    check(lib, lib.parseq_enc_attention(qkv.data_ptr(), B, T, D, heads, out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    q, k, v = qkv.float().reshape(B, T, 3, heads, d).permute(2, 0, 3, 1, 4)
    s = (q @ k.transpose(-1, -2)) * (d ** -0.5)
    e = torch.exp(s - s.max(-1, keepdim=True).values)
    o = (e.bfloat16().float() @ v) / e.sum(-1, keepdim=True)
    ref = o.permute(0, 2, 1, 3).reshape(B * T, D)
    err = (out.float() - ref).abs().max().item()
    assert err <= 2 ** -7 * ref.abs().max().item() + 1e-3, err
