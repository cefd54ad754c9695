"""The own FP64 DMMA GEMMs (gemm_backend 0) against cuBLAS ZGEMM (gemm_backend 1) around every edge of their tiles
(Gram 64 x 96, update 64 rows x 96 columns, 16 complex k per stage) and at the nonlocal shapes of the 128-atom Si
benchmark cell, with complex alpha and beta."""
import itertools
import pytest
import torch

pytestmark = pytest.mark.gpu

EDGES_M = [1, 15, 16, 17, 63, 64, 65]      # Gram rows / update rows (tile 64)
EDGES_N = [1, 15, 16, 17, 95, 96, 97]      # columns (tile 96)
ALPHA, BETA = 0.7 - 0.2j, -0.3 + 1.1j


def _rand(shape, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    from gpu_common import ctx
    return torch.view_as_complex(torch.randn(*shape, 2, generator=g, dtype=torch.float64)).to(ctx().device)


def _both(transA, A, B, C0, alpha, beta):
    """(own kernels, cuBLAS) results of C = alpha op(A) B + beta C0."""
    from gpu_common import ctx
    c = ctx()
    out = []
    for backend in (0, 1):
        c.set_option("gemm_backend", backend)
        try:
            out.append(c.zgemm(transA, A, B, C0.clone(), alpha, beta))
        finally:
            c.set_option("gemm_backend", 0)
    return out


def _rel(x, ref):
    return (x - ref).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize("m,n", list(itertools.product(EDGES_M, EDGES_N)))
def test_gram_tile_edges_match_cublas(m, n):
    K = 1001                                            # odd, not a multiple of the 16-deep stage
    A, B, C0 = _rand((m, K), 1), _rand((n, K), 2), _rand((n, m), 3)
    own, ref = _both("C", A, B, C0, ALPHA, BETA)
    assert _rel(own, ref) <= 1e-12


@pytest.mark.parametrize("rows,n", list(itertools.product(EDGES_M, EDGES_N)))
@pytest.mark.parametrize("k", [1, 15, 17, 33])
def test_update_tile_edges_match_cublas(rows, n, k):
    A, S, X0 = _rand((k, rows), 4), _rand((n, k), 5), _rand((n, rows), 6)
    own, ref = _both("N", A, S, X0, ALPHA, BETA)
    assert _rel(own, ref) <= 1e-12


def test_nonlocal_shapes_match_cublas():
    """P'psi (640 x 259 over 135 491 plane waves) and Hpsi += P (D P'psi) (135 491 x 259 over 640, beta = 1)."""
    npw, nproj, M = 135491, 640, 259
    P, psi = _rand((nproj, npw), 7), _rand((M, npw), 8)
    own, ref = _both("C", P, psi, torch.zeros((M, nproj), dtype=torch.complex128, device=P.device), ALPHA, 0.0)
    assert _rel(own, ref) <= 1e-12
    dproj, hpsi = _rand((M, nproj), 9), _rand((M, npw), 10)
    own, ref = _both("N", P, dproj, hpsi, 1.0, 1.0)
    assert _rel(own, ref) <= 1e-12
