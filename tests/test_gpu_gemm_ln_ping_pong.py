"""Boundaries of the persistent GEMM + LayerNorm kernel's partition (gemm_ln.cuh MODE 2): each CTA pair walks 64-row
tiles with the grid's stride, and its two MMA warpgroups take the pair's tiles in turn (ping-pong), so a pair's tile
count decides which warpgroup runs last.  The pair count is the one the launcher reports.  x must equal the unfused
GEMM's residual update, xn the full-row kernel's at K = 384."""
import pytest
import torch

from test_gpu_gemm_ln_persistent import D, _gemm_ln, _operands, _unfused_x

pytestmark = pytest.mark.gpu

CASES = {
    "one-tile": lambda n: 64,
    "one-partial-tile": lambda n: 40,
    "three-per-pair": lambda n: 64 * 3 * n,                 # odd: warpgroup 2 has one tile fewer
    "below-2x-pairs": lambda n: 64 * (2 * n - 1),
    "at-2x-pairs": lambda n: 64 * 2 * n,
    "above-2x-pairs": lambda n: 64 * (2 * n + 1),
    "last-tile-1-row": lambda n: 64 * 2 * n + 1,
    "last-tile-63-rows": lambda n: 64 * (3 * n - 1) + 63,
}


@pytest.fixture(scope="module")
def clusters(lib):
    A, W, bias, gamma, beta, x0 = _operands(1, 384, 0)
    _gemm_ln(lib, A, W, bias, x0, gamma, beta)
    n = lib.parseq_debug_int(None, b"ln_clusters")
    assert n > 0
    return n


@pytest.mark.parametrize("K", [384, 1536])
@pytest.mark.parametrize("case", list(CASES))
def test_ping_pong_partition(lib, clusters, case, K):
    M = CASES[case](clusters)
    A, W, bias, gamma, beta, x0 = _operands(M, K, 7 * M + K)
    x = x0.clone()
    xn = _gemm_ln(lib, A, W, bias, x, gamma, beta)
    assert torch.equal(x, _unfused_x(lib, A, W, bias, x0.clone()))
    ref_n = torch.nn.functional.layer_norm(x, (D,), gamma, beta, 1e-6)
    assert ((xn.float() - ref_n).abs() <= 2.0 ** -8 * ref_n.abs() + 1e-5).all()
    if K < 768:
        xf = x0.clone()
        xnf = _gemm_ln(lib, A, W, bias, xf, gamma, beta, ln_split=1)
        assert torch.equal(x, xf) and torch.equal(xn, xnf)
