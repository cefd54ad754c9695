"""The device XC kernel against the extended-precision reference and its host build, the XC potential as the functional
derivative of the XC energy through TermXc.potential, and a fully polarised SCF (run on an H100: -m gpu)."""
import math
import os
import numpy as np
import pytest
import torch

import xc_reference as xr
from test_xc_reference import (emu, run_emu, polarised_points, unpolarised_points, reference, magnitudes,  # noqa: F401
                               assert_close)
from upf_data import UPF_DIR, product_psp

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("functional", xr.FUNCTIONALS)
def test_device_sweep_matches_reference_and_host(emu, functional, n_spin):
    """The sweep of test_xc_reference on the device: the reference's bound, and the host build of the same bodies
    to 1e-13 relative (the device's FMA contraction and pow / cbrt differ from the host's at ulp level only)."""
    from dftk_b200 import xc as pxc
    from gpu_common import ctx, to_dev
    gga = functional.startswith("gga")
    rho, sigma = (unpolarised_points if n_spin == 1 else polarised_points)(gga)
    e, vr, vs = pxc.evaluate(ctx(), [functional], to_dev(rho), None if sigma is None else to_dev(sigma))
    e, vr = e.cpu().numpy(), vr.cpu().numpy()
    re, rvr, rvs = reference((functional,), rho, sigma)
    me, mr, ms = magnitudes(rho, sigma)
    assert_close(e, re, me, "e", rho, sigma)
    assert_close(vr, rvr, mr[None, :], "vrho", rho, sigma)
    he, hvr, hvs = run_emu(emu, (functional,), rho, sigma)
    # The correlation forms sum terms of order A ln(...) (A = 0.0311 Ha, the paramagnetic prefactor of PW92 and VWN)
    # that cancel towards a small eps_c at large rs, so an ulp of the device's log / atan against the host's is an ulp
    # of A: that size joins the scale here (VWN's vrho at rs ~ 3e3 differs by 1e-13 of eps_c alone).
    n = np.maximum(rho, 0.0).sum(axis=0)
    assert np.all(np.abs(e - he) <= 1e-13 * (np.abs(he) + me + 0.0311 * n))
    assert np.all(np.abs(vr - hvr) <= 1e-13 * (np.abs(hvr) + mr + 0.0311))
    if gga:
        vs = vs.cpu().numpy()
        assert_close(vs, rvs, ms[None, :], "vsigma", rho, sigma)
        assert np.all(np.abs(vs - hvs) <= 1e-13 * (np.abs(hvs) + ms))


DIAMOND = 6.74 * np.array([[0.0, 0.5, 0.5], [0.5, 0.0, 0.5], [0.5, 0.5, 0.0]])


def _xc_basis(functionals, n_spin, nlcc):
    import dftk_b200 as dftk
    if nlcc:
        atoms = [dftk.ElementPsp("C", psp=product_psp("C_m.upf"))] * 2
    else:
        atoms = [dftk.ElementPsp("Si", psp=dftk.load_psp(os.path.join(UPF_DIR, "Si-q4.gth")))] * 2
    kw = dict(magnetic_moments=[1.0, 0.5]) if n_spin == 2 else {}
    model = dftk.model_DFT(DIAMOND, atoms, [np.ones(3) / 8, -np.ones(3) / 8], functionals=list(functionals), **kw)
    basis = dftk.PlaneWaveBasis(model, Ecut=8, kgrid=(1, 1, 1))
    assert model.n_spin_components == n_spin
    assert (basis.term("Xc").rho_core is not None) == nlcc
    return basis


def _smooth(basis, modes, offset, amp, seed):
    """A band-limited real function on the FFT grid: offset + amp sum of low-frequency cosines."""
    nx, ny, nz = basis.fft_size
    i = np.arange(nx * ny * nz)
    x = np.stack([(i % nx) / nx, (i // nx % ny) / ny, (i // (nx * ny)) / nz])
    rng = np.random.default_rng(seed)
    f = np.full(i.size, float(offset))
    for _ in range(modes):
        k = rng.integers(-2, 3, 3)
        f += amp * rng.uniform(-1, 1) * np.cos(2 * math.pi * (k @ x) + rng.uniform(0, 2 * math.pi))
    return f


@pytest.mark.parametrize("nlcc", [False, True], ids=["hgh", "nlcc"])
@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("functionals", [("lda_x", "lda_c_pw"), ("gga_x_pbe", "gga_c_pbe")], ids=["lda", "pbe"])
def test_potential_is_energy_derivative(functionals, n_spin, nlcc):
    """(E[rho + h drho] - E[rho - h drho]) / 2h, Richardson-extrapolated in h, equals sum V drho dvol: pins the
    -2 div(vsigma grad rho) assembly (the 1/2 on sigma_ud, the (uu, ud, dd) packing, the sign of the divergence) and
    that the core density enters rho and grad rho while V stays the derivative with respect to rho."""
    basis = _xc_basis(functionals, n_spin, nlcc)
    term = basis.term("Xc")
    dev = basis.G_vectors_cart.device
    rho = np.stack([_smooth(basis, 6, 0.03 + 0.01 * s, 0.004, 10 + s) for s in range(n_spin)])
    drho = np.stack([_smooth(basis, 6, 0.0, 1.0, 20 + s) for s in range(n_spin)])
    rho_t = torch.tensor(rho, dtype=torch.float64, device=dev)
    drho_t = torch.tensor(drho, dtype=torch.float64, device=dev)
    _, V = term.potential(basis, rho_t)
    predicted = float((V * drho_t).sum()) * basis.dvol

    def central(h):
        return (term.potential(basis, rho_t + h * drho_t)[0] - term.potential(basis, rho_t - h * drho_t)[0]) / (2 * h)
    h = 1e-4
    d1, d2 = central(h), central(h / 2)
    fd = (4 * d2 - d1) / 3
    assert abs(d1 - d2) > 0 or abs(predicted) < 1e-12
    # The core density carries content up to the grid's Nyquist frequencies, where the FFT gradient of a real field is
    # not exactly the adjoint of the FFT divergence; a band-limited rho has none.  The gap this leaves was 1.8e-8
    # relative for PBE, n_spin = 1 (this test's setup, on an H100 SXM at its default power limit); the bound is 1e-7.
    assert abs(fd - predicted) <= (1e-7 if nlcc else 1e-8) * abs(predicted)



@pytest.fixture(scope="module")
def hydrogen():
    """One electron, spin-polarised (moment 1, T = 1e-3 Ha), in an 8 bohr cube at Ecut 15 Ha: the device SCF and the
    oracle's, per functional set, run once for the tests below."""
    cache = {}

    def run(tag):
        if tag in cache:
            return cache[tag]
        import dftk_b200 as dftk
        from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
        from oracle.psp_hgh import PspHgh
        from oracle import nlcc
        funs = ("lda_x", "lda_c_pw") if tag == "lda" else ("gga_x_pbe", "gga_c_pbe")
        path = os.path.join(UPF_DIR, f"H-{tag}-q1.hgh")
        lattice = 8.0 * np.eye(3)
        pm = dftk.model_DFT(lattice, [dftk.ElementPsp("H", psp=dftk.load_psp(path))], [np.zeros(3)],
                            functionals=list(funs), magnetic_moments=[1.0], temperature=1e-3)
        with open(path) as fh:
            opsp = PspHgh.parse(fh.read())
        opsp.Z = 1                       # the file carries only the valence charge
        om = Model(lattice, [Element("H", opsp)], [np.zeros(3)], functionals=funs, magnetic_moments=[1.0],
                   temperature=1e-3)
        basis = dftk.PlaneWaveBasis(pm, Ecut=15, kgrid=(1, 1, 1))
        res = dftk.self_consistent_field(basis, tol=1e-9)
        ob = OBasis(om, 15, kgrid=(1, 1, 1))
        ores = nlcc.self_consistent_field(ob, tol=1e-9)
        cache[tag] = (basis, res, ob, ores)
        return cache[tag]
    return run


def _oracle_eigenvalues(basis, ob, ores, spin, n):
    jk = [j for j, k in enumerate(ob.kpoints) if k.spin == spin][0]
    return np.asarray(ores["eigenvalues"][jk][:n])


@pytest.mark.parametrize("tag", ["lda", "pbe"])
def test_fully_polarised_hydrogen_scf(hydrogen, tag):
    """rho_dn vanishes, so every minority point sits at the fully polarised edge.  The device SCF converges to the
    oracle's energy and density, and the spectrum of its final Hamiltonian (re-diagonalised tightly) matches the
    oracle's in both spin channels: the minority levels are finite, above the majority ones and within a few Ha of
    them, which a minority potential taken from the unscreened edge (vrho_dn of hundreds of Ha) would not give."""
    from dftk_b200.scf import FixedBands, next_density
    basis, res, ob, ores = hydrogen(tag)
    assert res["converged"] and ores["converged"]
    assert ob.fft_size == basis.fft_size
    rho = res["rho"].cpu().numpy()
    assert np.abs(rho[1]).max() < 1e-10 * rho[0].max()
    assert abs(res["energies"].total - ores["energies"]["total"]) < 1e-8
    assert np.linalg.norm(rho - ores["rho"]) * math.sqrt(basis.dvol) < 1e-7
    tight = next_density(res["ham"], FixedBands(4, 8), tol=1e-10, maxiter=400)
    eig = {}
    for ik, kpt in enumerate(basis.kpoints):
        eig[kpt.spin] = np.asarray(tight["eigenvalues"][ik])[:4]
        np.testing.assert_allclose(eig[kpt.spin], _oracle_eigenvalues(basis, ob, ores, kpt.spin, 4), atol=1e-6)
    assert np.all(np.isfinite(eig[1]))
    assert eig[0][0] < eig[1][0] < eig[0][0] + 3.0


@pytest.mark.xfail(strict=False, reason=(
    "the batched device LOBPCG does not hold the empty minority block converged once the SCF's diagonalisation "
    "tolerance falls below ~1e-8: the block ends unconverged (at or before maxiter) and its returned eigenvalues are "
    "off by 7e-5 Ha (LDA) to 0.1-1.3 Ha (PBE), varying from run to run, while a fresh tight solve of the same "
    "Hamiltonian matches the oracle (test_fully_polarised_hydrogen_scf)"))
@pytest.mark.parametrize("tag", ["lda", "pbe"])
def test_fully_polarised_hydrogen_scf_eigenvalues(hydrogen, tag):
    """The eigenvalues the SCF itself returns, in both spin channels, against the oracle's."""
    basis, res, ob, ores = hydrogen(tag)
    assert res["converged"]
    for ik, kpt in enumerate(basis.kpoints):
        np.testing.assert_allclose(np.asarray(res["eigenvalues"][ik])[:2], _oracle_eigenvalues(basis, ob, ores, kpt.spin, 2),
                                   atol=1e-6)
