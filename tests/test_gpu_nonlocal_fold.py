"""The folded nonlocal apply (blas.cu: kb_apply_nonlocal_folded, real-A products k_rgemm_cn / k_rgemm_nn) against the
complex cuBLAS products (gemm_backend 1) on Γ and time-reversal-invariant k-blocks, with and without accumulation.
The launch count tells which path ran: six launches per band chunk folded (fold, Gram, split-K reduce, D, update,
unfold), four on the complex path (Gram, reduce, D, update).  A non-TRIM block and a block with random projectors
must keep the complex path."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-13
BANDS = [1, 15, 16, 17, 63, 64, 65, 95, 96, 97, 259]
FOLDED, COMPLEX = 6, 4
A_SI = 10.26 / 2


def _supercell(rep):
    lat = rep * np.array([[0, A_SI, A_SI], [A_SI, 0, A_SI], [A_SI, A_SI, 0]])
    pos = [(b + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep)
           for b in (np.ones(3) / 8, -np.ones(3) / 8)]
    return lat, pos


def _blocks(rep, Ecut, kcoords):
    import dftk_b200 as dftk
    lat, pos = _supercell(rep)
    Si = dftk.ElementPsp("Si")
    model = dftk.model_DFT(lat, [Si] * len(pos), pos, functionals=dftk.LDA(), symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=dftk.ExplicitKpoints(kcoords))
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=dftk.guess_density(basis))
    return basis, [blk.bind() for blk in ham]


def _crand(g, *shape):
    return torch.view_as_complex(torch.randn(*shape, 2, generator=g, dtype=torch.float64)).to("cuda")


def _apply(kb, psi, out0, backend, accumulate):
    c = kb.ctx
    c.set_option("gemm_backend", backend)
    try:
        out = out0.clone()
        c.launch_count(reset=True)
        kb.apply_terms(psi, 4, out=out, accumulate=accumulate)
        torch.cuda.synchronize()
        return out, c.launch_count()
    finally:
        c.set_option("gemm_backend", 0)


def _check(kb, nb, launches, seed=0):
    g = torch.Generator().manual_seed(seed)
    psi, out0 = _crand(g, nb, kb.n_pw), _crand(g, nb, kb.n_pw)
    for accumulate in (False, True):
        ref, _ = _apply(kb, psi, out0, 1, accumulate)
        got, n = _apply(kb, psi, out0, 0, accumulate)
        err = ((got - ref).abs().max() / ref.abs().max()).item()
        assert err <= TOL, (nb, accumulate, err)
        assert n == launches, (nb, n)


@pytest.fixture(scope="module")
def si16():
    basis, kbs = _blocks(2, 15.0, [[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [0.1, -0.2, 0.3]])
    return basis, kbs


@pytest.mark.parametrize("nb", BANDS)
def test_gamma_block_band_edges(si16, nb):
    _check(si16[1][0], nb, FOLDED, seed=nb)


def test_trim_block(si16):
    _check(si16[1][1], 17, FOLDED)
    _check(si16[1][1], 97, FOLDED)


def test_non_trim_block_keeps_complex_path(si16):
    _check(si16[1][2], 17, COMPLEX)


@pytest.mark.parametrize("n_proj", [1, 15, 16, 17, 63, 64, 65])
def test_projector_count_edges(si16, n_proj):
    import dftk_b200
    basis, kbs = si16
    kpt = basis.kpoints[0]
    op = basis.term("AtomicNonlocal").ops[0]
    assert op.P.shape[0] >= n_proj
    P = op.P[:n_proj].contiguous()
    D = np.asarray(op.D.cpu() if torch.is_tensor(op.D) else op.D)[:n_proj, :n_proj]
    kb = dftk_b200.KBlock(basis.fft_grid, kpt.mapping.cpu().numpy(), P=P, D=D)
    _check(kb, 65, FOLDED, seed=n_proj)


def test_random_projectors_keep_complex_path(si16):
    import dftk_b200
    basis, kbs = si16
    kpt = basis.kpoints[0]
    g = torch.Generator().manual_seed(3)
    P = _crand(g, 20, kpt.n_G)
    D = np.eye(20)
    kb = dftk_b200.KBlock(basis.fft_grid, kpt.mapping.cpu().numpy(), P=P, D=D)
    _check(kb, 33, COMPLEX)


def test_band_energies_folded(si16):
    kb = si16[1][0]
    g = torch.Generator().manual_seed(5)
    psi = _crand(g, 40, kb.n_pw)
    c = kb.ctx
    c.set_option("gemm_backend", 1)
    try:
        _, en_ref = kb.band_energies(psi)
    finally:
        c.set_option("gemm_backend", 0)
    _, en = kb.band_energies(psi)
    np.testing.assert_allclose(en, en_ref, rtol=1e-12, atol=1e-13 * np.abs(en_ref).max())


def test_wide_block_is_chunked(si16):
    """777 columns (a LOBPCG [X P R] block) run as three chunks of 259."""
    _check(si16[1][0], 777, 3 * FOLDED)


def test_benchmark_cell():
    """Γ block of the 128-atom Si cell at Ecut 30 (n_pw 135 491, 640 projectors), 259 bands."""
    basis, kbs = _blocks(4, 30.0, [[0.0, 0.0, 0.0]])
    kb = kbs[0]
    assert kb.n_pw == 135491 and kb.n_proj == 640
    _check(kb, 259, FOLDED)
