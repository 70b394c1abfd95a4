"""The GEMM's bf16 epilogues (gemm.cuh): tiles staged in swizzled shared memory and stored by TMA where the output is
a valid tensor map, register stores where it is not (misaligned base or row pitch).  Both must give the same bits, and
the bf16 output must be the round-to-nearest-even of the fp32 epilogue's output."""
import pytest
import torch

pytestmark = pytest.mark.gpu

K = 384


def _run(lib, A, W, bias, mode, out, ldo, alpha=1.0, resid=None):
    from parseq_b200.engine import check
    M = A.shape[0]
    N = W.shape[0]
    check(lib, lib.parseq_gemm_bf16(A.data_ptr(), A.stride(0), W.data_ptr(), W.stride(0), bias.data_ptr(), M, N, K, mode,
                                    alpha, resid.data_ptr() if resid is not None else None,
                                    resid.stride(0) if resid is not None else 0, 0, out.data_ptr(), ldo,
                                    torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out


def _operands(M, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn((M, K), device="cuda", generator=g).bfloat16()
    W = (torch.randn((N, K), device="cuda", generator=g) * 0.05).bfloat16()
    bias = torch.randn((N,), device="cuda", generator=g)
    return A, W, bias


def _misaligned(M, N):
    """A [M, N] bf16 view whose base is 2 bytes past a 16-B boundary, with an odd row pitch (N + 1)."""
    buf = torch.zeros(M * (N + 1) + 8, device="cuda", dtype=torch.bfloat16)
    return buf[1:1 + M * (N + 1)].view(M, N + 1)[:, :N], N + 1


@pytest.mark.parametrize("N", [95, 576, 768, 1152, 1536])
@pytest.mark.parametrize("M", [1, 130, 8192 + 77, 65536])
def test_bf16_is_rounded_fp32_epilogue(lib, M, N):
    """Ragged M and N (TMA clipping at the tensor map's bounds): bf16 output == RNE(fp32 output), bit for bit."""
    A, W, bias = _operands(M, N, M + N)
    for alpha in (1.0, 0.125):
        f32 = _run(lib, A, W, bias, 0, torch.empty((M, N), device="cuda"), N, alpha)
        guard = torch.full((M + 1, N), -7.0, device="cuda", dtype=torch.bfloat16)   # a row past M must stay untouched
        bf = _run(lib, A, W, bias, 1, guard, N, alpha)[:M]
        assert torch.equal(bf.view(torch.int16), f32.bfloat16().view(torch.int16))
        assert bool((guard[M] == -7.0).all())
    ref = A.float() @ W.float().t() + bias
    assert (f32 * 8.0 - ref).abs().max().item() <= 2e-4 * ref.abs().max().item()


@pytest.mark.parametrize("M,N", [(130, 1536), (8192 + 77, 1152), (65536, 1536)])
def test_gelu_against_torch_and_store_paths(lib, M, N):
    """GELU (ex2.approx polynomial, not reproducible in torch): within one bf16 ulp of torch's GELU, and the TMA-store
    and register-store paths (misaligned output) give the same bits, for the plain bf16 epilogue too; every block_n /
    cta_group setting as well."""
    from parseq_b200.engine import check
    A, W, bias = _operands(M, N, 3 * M + N)
    acc = A.float() @ W.float().t() + bias
    ref = torch.nn.functional.gelu(acc)
    for mode in (1, 2):
        tma = _run(lib, A, W, bias, mode, torch.empty((M, N), device="cuda", dtype=torch.bfloat16), N)
        if mode == 2:
            assert (tma.float() - ref).abs().max().item() <= 2 ** -7 * ref.abs().max().item()
            assert (tma.float() == ref.bfloat16().float()).float().mean().item() > 0.99
        out, ldo = _misaligned(M, N)
        reg = _run(lib, A, W, bias, mode, out, ldo)
        assert torch.equal(reg.view(torch.int16), tma.view(torch.int16))
        try:
            for cg, bn in [(1, 64), (1, 192), (1, 256), (2, 128), (2, 256)]:
                check(lib, lib.parseq_set_option(None, b"cta_group", cg))
                check(lib, lib.parseq_set_option(None, b"block_n", bn))
                v = _run(lib, A, W, bias, mode, torch.empty((M, N), device="cuda", dtype=torch.bfloat16), N)
                assert torch.equal(v.view(torch.int16), tma.view(torch.int16)), (cg, bn)
        finally:
            check(lib, lib.parseq_set_option(None, b"cta_group", 0))
            check(lib, lib.parseq_set_option(None, b"block_n", 0))


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N", [1152, 1536])
def test_repeated_launches_bit_identical(lib, N, mode):
    """M = 65536: 4608 / 6144 tiles, ~35-47 per CTA, so each warpgroup reuses its staging tile ~20 times per launch."""
    M = 65536
    A, W, bias = _operands(M, N, N + mode)
    outs = []
    for _ in range(3):
        if mode == 0:
            x = torch.ones((M, N), device="cuda")
            outs.append(_run(lib, A, W, bias, 0, x, N, resid=x).clone())
        else:
            outs.append(_run(lib, A, W, bias, mode, torch.empty((M, N), device="cuda", dtype=torch.bfloat16), N).clone())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
