"""The persistent column-split GEMM + LayerNorm kernel (gemm_ln.cuh MODE 2, the default at D = 384): clusters of two CTAs
walk 128-row tiles with the grid's stride (one cluster per SM pair), the producer runs ahead across tiles and fetches
each tile's x slice into shared memory.  Tile counts below, equal to and far above the number of clusters, ragged last
tiles, both K of the encoder (attn.proj: two 192-column row-statistics parts, fc2: four 96-column parts)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

D = 384


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _clusters():
    return torch.cuda.get_device_properties(0).multi_processor_count // 2


def _operands(M, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((D, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((D,), device="cuda", generator=g)
    gamma = 1.0 + 0.1 * torch.randn((D,), device="cuda", generator=g)
    beta = 0.05 * torch.randn((D,), device="cuda", generator=g)
    x0 = torch.randn((M, D), device="cuda", generator=g) + 0.3 * torch.randn((M, 1), device="cuda", generator=g)
    return A, W, bias, gamma, beta, x0


def _gemm_ln(lib, A, W, bias, x, gamma, beta, ln_split=0, pair_pdl=0):
    """x += A W^T + bias in place; returns xn.  A guard row past M in both outputs must stay untouched."""
    from parseq_b200.engine import check
    M, K = A.shape
    xg = torch.cat([x, torch.full((1, D), -3.0, device="cuda")])
    xn = torch.full((M + 1, D), -5.0, dtype=torch.bfloat16, device="cuda")
    try:
        check(lib, lib.parseq_set_option(None, b"ln_split", ln_split))
        check(lib, lib.parseq_set_option(None, b"pair_pdl", pair_pdl))
        check(lib, lib.parseq_gemm_ln_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, D, K, xg.data_ptr(),
                                           gamma.data_ptr(), beta.data_ptr(), 1e-6, xn.data_ptr(), _stream()))
        torch.cuda.synchronize()
    finally:
        check(lib, lib.parseq_set_option(None, b"ln_split", 0))
        check(lib, lib.parseq_set_option(None, b"pair_pdl", 0))
    assert bool((xg[M] == -3.0).all()) and bool((xn[M] == -5.0).all())
    x.copy_(xg[:M])
    return xn[:M]


def _unfused_x(lib, A, W, bias, x):
    """The GEMM's fp32 residual-accumulate epilogue, in place."""
    from parseq_b200.engine import check
    M, K = A.shape
    check(lib, lib.parseq_gemm_bf16(A.data_ptr(), K, W.data_ptr(), K, bias.data_ptr(), M, D, K, 0, 1.0, x.data_ptr(), D, 0,
                                    x.data_ptr(), D, _stream()))
    torch.cuda.synchronize()
    return x


def _sizes():
    c = _clusters()
    return [1, 77, 128 * c - 50, 128 * c, 128 * c + 1, 65536 + 77]


@pytest.mark.parametrize("K", [384, 1536])
@pytest.mark.parametrize("which", range(6), ids=["M1", "M77", "below", "equal", "one-more", "far-above"])
def test_persistent_gemm_ln(lib, which, K):
    M = _sizes()[which]
    A, W, bias, gamma, beta, x0 = _operands(M, K, M + K)
    x = x0.clone()
    xn = _gemm_ln(lib, A, W, bias, x, gamma, beta)
    # x: the k order of the unfused GEMM, then (acc + b) + x
    assert torch.equal(x, _unfused_x(lib, A, W, bias, x0.clone()))
    # xn: one bf16 rounding of the LayerNorm of the kernel's own x
    ref_n = torch.nn.functional.layer_norm(x, (D,), gamma, beta, 1e-6)
    assert ((xn.float() - ref_n).abs() <= 2.0 ** -8 * ref_n.abs() + 1e-5).all()
    if K < 768:
        # attn.proj: the row statistics in the order of the full-row kernel
        xf = x0.clone()
        xnf = _gemm_ln(lib, A, W, bias, xf, gamma, beta, ln_split=1)
        assert torch.equal(x, xf) and torch.equal(xn, xnf)
    # deterministic, and the same bits with programmatic dependent launch on the pair launch
    for pdl in (0, 1):
        x2 = x0.clone()
        xn2 = _gemm_ln(lib, A, W, bias, x2, gamma, beta, ln_split=2, pair_pdl=pdl)
        assert torch.equal(x, x2) and torch.equal(xn, xn2)
