"""The Teter-Pade and Perdew-Zunger LDAs and the PBEsol, revPBE and RPBE GGAs on the device (run on an H100: -m gpu):
the kernel against the extended-precision reference and its host build, TermXc.potential as the derivative of the XC
energy, the reference's iron LDA SCF against ABINIT, and SCFs and NLCC forces against the oracle."""
import math
import numpy as np
import pytest
import torch

import xc_reference_families as xrf
import xc_oracle_families
from test_xc_reference import magnitudes, assert_close
from test_xc_families import (emu, run_emu, reference, sweep_points, SETS, SET_IDS,  # noqa: F401
                              iron_lda_reference, IRON_LATTICE, IRON_LDA_PSP,
                              assert_iron_lda_matches_abinit)
from test_gpu_xc_reference import test_potential_is_energy_derivative as potential_is_energy_derivative
from test_gpu_xc_reference import _xc_basis, _smooth
from test_gpu_scf import _compare_scf
from test_gpu_upf import _models, _scf_pair, _compare, DIAMOND, FCC_AL
from silicon import LATTICE, POSITIONS

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("functional", xrf.FUNCTIONALS)
def test_device_sweep_matches_reference_and_host(emu, functional, n_spin):
    """The sweep on the device: the reference's bound, and the host build of the same bodies to 1e-13 relative, with
    the scales of test_gpu_xc_reference (the correlation's A ln(...) terms join the scale of e and vrho)."""
    from dftk_b200 import xc as pxc
    from gpu_common import ctx, to_dev
    rho, sigma = sweep_points(functional, n_spin)
    e, vr, vs = pxc.evaluate(ctx(), [functional], to_dev(rho), None if sigma is None else to_dev(sigma))
    e, vr = e.cpu().numpy(), vr.cpu().numpy()
    re, rvr, rvs = reference((functional,), rho, sigma)
    me, mr, ms = magnitudes(rho, sigma)
    assert_close(e, re, me, "e", rho, sigma)
    assert_close(vr, rvr, mr[None, :], "vrho", rho, sigma)
    he, hvr, hvs = run_emu(emu, (functional,), rho, sigma)
    n = np.maximum(rho, 0.0).sum(axis=0)
    assert np.all(np.abs(e - he) <= 1e-13 * (np.abs(he) + me + 0.0311 * n))
    assert np.all(np.abs(vr - hvr) <= 1e-13 * (np.abs(hvr) + mr + 0.0311))
    if sigma is not None:
        vs = vs.cpu().numpy()
        assert_close(vs, rvs, ms[None, :], "vsigma", rho, sigma)
        assert np.all(np.abs(vs - hvs) <= 1e-13 * (np.abs(hvs) + ms))


@pytest.mark.parametrize("nlcc", [False, True], ids=["hgh", "nlcc"])
@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("functionals", SETS[:4], ids=SET_IDS[:4])
def test_potential_is_energy_derivative(functionals, n_spin, nlcc):
    """The check of test_gpu_xc_reference, with its bounds, for the new functional sets: the Richardson-extrapolated
    finite difference of the XC energy along a smooth direction equals sum V drho dvol."""
    potential_is_energy_derivative(functionals, n_spin, nlcc)


@pytest.mark.parametrize("nlcc,offset", [(False, 0.03), (False, 0.5), (True, 0.5)], ids=["hgh-rs>1", "hgh-rs<1", "nlcc-rs<1"])
@pytest.mark.parametrize("n_spin", [1, 2])
def test_perdew_zunger_potential_is_energy_derivative(n_spin, nlcc, offset):
    """The same check for Slater + Perdew-Zunger, with the density on one side of rs = 1.  PZ's two branches do not
    meet there (eps_c = -0.0596 below, -0.059632 above), so E jumps wherever rho crosses rs = 1 (n = 0.2387), and a
    finite difference across that, as the core density of C_m.upf forces at the densities of the check above, measures
    the jump (5.6e-4 relative on an H100 at n_spin = 1).  At a mean density of 0.03 every point has rs > 1; at 0.5,
    core density or not, every point has rs < 1."""
    basis = _xc_basis(("lda_x", "lda_c_pz"), n_spin, nlcc)
    term = basis.term("Xc")
    dev = basis.G_vectors_cart.device
    rho = np.stack([_smooth(basis, 6, offset + 0.01 * s, 0.004, 10 + s) for s in range(n_spin)])
    drho = np.stack([_smooth(basis, 6, 0.0, 1.0, 20 + s) for s in range(n_spin)])
    rho_t = torch.tensor(rho, dtype=torch.float64, device=dev)
    drho_t = torch.tensor(drho, dtype=torch.float64, device=dev)
    tot = rho_t.sum(0) + (0 if term.rho_core is None else term.rho_core.sum(0))
    rs = (3 / (4 * math.pi * tot)) ** (1 / 3)
    assert bool((rs > 1.01).all()) if offset < 0.1 else bool((rs < 0.99).all())
    _, V = term.potential(basis, rho_t)
    predicted = float((V * drho_t).sum()) * basis.dvol

    def central(h):
        return (term.potential(basis, rho_t + h * drho_t)[0] - term.potential(basis, rho_t - h * drho_t)[0]) / (2 * h)
    d1, d2 = central(1e-4), central(5e-5)
    fd = (4 * d2 - d1) / 3
    assert abs(d1 - d2) > 0
    assert abs(fd - predicted) <= (1e-7 if nlcc else 1e-8) * abs(predicted)


def test_unknown_functional_raises():
    import dftk_b200 as dftk
    from dftk_b200 import xc as pxc
    from gpu_common import ctx, to_dev
    with pytest.raises(NotImplementedError):
        pxc.evaluate(ctx(), ["gga_x_b88"], to_dev(np.full((1, 4), 0.1)), to_dev(np.full((1, 4), 0.01)))
    assert dftk.PBEsol() == ["gga_x_pbe_sol", "gga_c_pbe_sol"]


def test_iron_lda_vs_abinit():
    # reference: test/iron_lda.jl (bcc Fe, GTH-PADE-q8, lda_xc_teter93, collinear spin, T = 0.01, Ecut 15, fft 20,
    # shifted 4x4x4 grid; ABINIT eigenvalues and E_tot to 5e-6)
    import dftk_b200 as dftk
    ref = iron_lda_reference()
    Fe = dftk.ElementPsp("Fe", psp=dftk.load_psp(IRON_LDA_PSP))
    assert Fe.psp.Zion == 8
    model = dftk.model_DFT(IRON_LATTICE, [Fe], [[0, 0, 0]], functionals=["lda_xc_teter93"], temperature=0.01,
                           magnetic_moments=[4.0])
    basis = dftk.PlaneWaveBasis(model, Ecut=15, kgrid=dftk.MonkhorstPack((4, 4, 4), kshift=(0.5, 0.5, 0.5)),
                                fft_size=(20, 20, 20))
    assert len(basis.kpoints) == 12
    res = dftk.self_consistent_field(basis, rho=dftk.guess_density(basis, [4.0]), mixing=dftk.KerkerMixing(),
                                     is_converged=dftk.ScfConvergenceEnergy(1e-10),
                                     nbandsalg=dftk.AdaptiveBands(model, n_bands_converge=8))
    assert_iron_lda_matches_abinit(basis.kpoints, res["eigenvalues"], res["energies"].total, ref)


# ------------------------------------------------------------------ against the oracle (BASELINE tolerances)
@pytest.mark.parametrize("functionals", [None, ("lda_x", "lda_c_pz")], ids=["pbesol", "pz"])
def test_silicon_with_symmetries_matches_oracle(monkeypatch, functionals):
    """Si2 with its 48 symmetries on a 3x3x3 grid, PBEsol() (None) or Slater + Perdew-Zunger."""
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle import scf as oscf
    xc_oracle_families.install(monkeypatch)
    funs = dftk.PBEsol() if functionals is None else list(functionals)
    Si = dftk.ElementPsp("Si", functional="lda")
    model = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=funs)
    assert len(model.symmetries) == 48
    basis = dftk.PlaneWaveBasis(model, Ecut=12, kgrid=(3, 3, 3))
    res = dftk.self_consistent_field(basis, tol=1e-9)
    assert res["converged"]
    om = Model(LATTICE, [Element("Si")] * 2, POSITIONS, functionals=tuple(funs))
    ob = OBasis(om, 12, kgrid=(3, 3, 3))
    assert ob.fft_size == basis.fft_size and len(ob.kpoints) == len(basis.kpoints)
    ores = oscf.self_consistent_field(ob, tol=1e-9)
    _compare_scf(res, ores, basis, ob, 2, 4)


def test_carbon_collinear_rpbe_nlcc_matches_oracle(monkeypatch):
    xc_oracle_families.install(monkeypatch)
    dftk, pm, om = _models("C_m.upf", DIAMOND, [np.ones(3) / 8, -np.ones(3) / 8], ("gga_x_rpbe", "gga_c_pbe"),
                           magnetic_moments=[1.0, 1.0], temperature=0.01)
    basis, res, ob, ores = _scf_pair(dftk, pm, om, 10, (1, 1, 1))
    assert pm.n_spin_components == 2 and basis.term("Xc").rho_core is not None
    _compare(basis, res, ob, ores, 2, 4)


def test_aluminium_revpbe_smearing_nlcc_matches_oracle(monkeypatch):
    xc_oracle_families.install(monkeypatch)
    dftk, pm, om = _models("Al_m.upf", FCC_AL, [np.zeros(3)], ("gga_x_pbe_r", "gga_c_pbe"), temperature=0.01)
    basis, res, ob, ores = _scf_pair(dftk, pm, om, 10, (3, 3, 3))
    _compare(basis, res, ob, ores, 1, 2)


def test_nlcc_forces_pbesol_match_oracle(monkeypatch):
    """test_gpu_upf.test_nlcc_forces_match_oracle with PBEsol: the same psi, occupation and rho on both sides (the
    oracle's SCF of a displaced C2 cell), every force term to 1e-10."""
    from oracle.basis import PlaneWaveBasis as OBasis
    from oracle import nlcc
    xc_oracle_families.install(monkeypatch)
    pos = [np.ones(3) / 8 + np.array([0.012, -0.006, 0.004]), -np.ones(3) / 8]
    dftk, pm, om = _models("C_m.upf", DIAMOND, pos, ("gga_x_pbe_sol", "gga_c_pbe_sol"), symmetries=False)
    ob = OBasis(om, 10, kgrid=(1, 1, 1))
    ores = nlcc.self_consistent_field(ob, tol=1e-10, maxiter=80)
    assert ores["converged"]
    ototal, oparts = nlcc.compute_forces(ob, ores["psi"], ores["occupation"], ores["rho"])
    basis = dftk.PlaneWaveBasis(pm, Ecut=10, kgrid=(1, 1, 1), fft_size=ob.fft_size)
    dev = basis.architecture.device
    psi = [torch.from_numpy(np.ascontiguousarray(ores["psi"][0].T)).to(dev)]
    rho = torch.from_numpy(ores["rho"]).to(dev)
    total, parts = dftk.compute_forces(basis, psi, ores["occupation"], rho=rho, per_term=True)
    assert set(parts) == {"AtomicLocal", "AtomicNonlocal", "Ewald", "Xc"}
    assert np.linalg.norm(np.array(parts["Xc"])) > 1e-3
    for name in parts:
        np.testing.assert_allclose(np.array(parts[name]), np.array(oparts[name]), atol=1e-10, err_msg=name)
    np.testing.assert_allclose(np.array(total), np.array(ototal), atol=1e-10)
