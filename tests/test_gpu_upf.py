"""GPU parity of the UPF path: the radial-transform kernel (dftk_b200_radial_transform) against the oracle's scipy-based
transforms, the form factors of a UPF basis, SCF with non-linear core correction, and the NLCC force."""
import math
import os
import numpy as np
import pytest
import torch

from silicon import LATTICE, POSITIONS
from upf_data import UPF_DIR as UPF, product_psp, oracle_psp

pytestmark = pytest.mark.gpu

FILES = ["Si.pbe-hgh.upf", "Tl.pbe-d-hgh.upf", "Al_m.upf", "C_m.upf"]
# special points and a dense grid up to 20 bohr^-1; 1041 values in all, not a multiple of the 128-thread block
Q = np.concatenate([[0.0, 1e-16, 1e-8, 1e-3], np.linspace(0.0, 20.0, 1037)])
DIAMOND = 6.74 / 2 * np.array([[0.0, 1, 1], [1, 0, 1], [1, 1, 0]])
FCC_AL = 7.65 / 2 * np.array([[0.0, 1, 1], [1, 0, 1], [1, 1, 0]])


def _dev():
    return torch.device("cuda:0")


def _both(name):
    return product_psp(name), oracle_psp(name)


@pytest.mark.parametrize("name", FILES)
def test_kernel_matches_oracle_for_every_function(name):
    prod, orc = _both(name)
    q = torch.from_numpy(Q).to(_dev())
    F = prod.radial_transform("proj", q).cpu().numpy()
    row = 0
    for l in range(orc.lmax + 1):
        for i in range(1, orc.n_proj_radial(l) + 1):
            ref = orc.eval_projector_fourier(i, l, Q)
            assert np.abs(F[row] - ref).max() <= 1e-12 * np.abs(ref).max(), (l, i)
            np.testing.assert_array_equal(prod.eval_psp_projector_fourier(i, l, q).cpu().numpy(), F[row])
            row += 1
    assert row == F.shape[0]
    checks = [(prod.eval_psp_local_fourier, orc.eval_local_fourier)]
    if orc.has_core_density:
        checks.append((prod.eval_psp_core_density_fourier, orc.eval_core_density_fourier))
    if orc.has_valence_density:
        checks.append((prod.eval_psp_valence_density_fourier, orc.eval_valence_density_fourier))
    for fp, fo in checks:
        got, ref = fp(q).cpu().numpy(), fo(Q)
        assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max(), fp.__name__


def test_kernel_on_synthetic_tables():
    """The ABI on its own: 17 functions (two launches of at most 16), every l, a log mesh with an odd and a uniform mesh
    with an even number of points, against 4π/q^l Σ g j_l(q r) from scipy."""
    from scipy.special import spherical_jn
    import dftk_b200 as dftk
    from dftk_b200.device import _ptr
    from dftk_b200.pseudo import _radial_ctx
    rng = np.random.default_rng(5)
    for r in (1e-5 * 1.0125 ** np.arange(1000), np.linspace(0.0, 8.0, 801)):
        n_f = 17
        ls = rng.integers(0, 4, n_f).astype(np.int32)
        ls[:4] = [0, 1, 2, 3]
        g = rng.standard_normal((n_f, len(r))) * np.exp(-r)[None, :] * r[None, :] ** 2
        g[3, 500:] = 0.0                                   # a function shorter than the mesh
        q = torch.from_numpy(Q).to(_dev())
        out = torch.empty((n_f, len(Q)), dtype=torch.float64, device=_dev())
        rd, gd = torch.from_numpy(r).to(_dev()), torch.from_numpy(np.ascontiguousarray(g)).to(_dev())
        h = _radial_ctx(_dev())
        dftk._lib.check(dftk._lib.lib().dftk_b200_radial_transform(h, len(r), _ptr(rd), n_f, _ptr(gd), _ptr(ls), len(Q),
                                                                   _ptr(q), _ptr(out)), h)
        F = out.cpu().numpy()
        for f in range(n_f):
            l = int(ls[f])
            ref = np.empty(len(Q))
            small = Q <= 10 * np.finfo(float).eps
            ref[small] = 4 * math.pi * np.sum(g[f] * r ** l) / [1, 3, 15, 105][l]
            qq = Q[~small]
            ref[~small] = 4 * math.pi * (spherical_jn(l, qq[:, None] * r[None, :]) @ g[f]) / qq ** l
            assert np.abs(F[f] - ref).max() <= 1e-12 * np.abs(ref).max(), (f, l)
        bad = ls.copy()
        bad[0] = 4
        assert dftk._lib.lib().dftk_b200_radial_transform(h, len(r), _ptr(rd), n_f, _ptr(gd), _ptr(bad), len(Q), _ptr(q),
                                                          _ptr(out)) != 0


def _models(name, lattice, positions, functionals, **kw):
    """(product model, oracle model) of one species."""
    import dftk_b200 as dftk
    from oracle.basis import Element, Model
    prod, orc = _both(name)
    sym = orc.element
    pm = dftk.model_DFT(lattice, [dftk.ElementPsp(sym, psp=prod)] * len(positions), positions, functionals=list(functionals),
                        **kw)
    okw = dict(kw)
    if "magnetic_moments" in okw:
        okw["magnetic_moments"] = list(okw["magnetic_moments"])
    om = Model(lattice, [Element(sym, orc)] * len(positions), positions, functionals=tuple(functionals), **okw)
    return dftk, pm, om


@pytest.mark.parametrize("name,lattice,positions", [
    ("C_m.upf", DIAMOND, [np.ones(3) / 8 + 0.01, -np.ones(3) / 8]),
    ("Al_m.upf", FCC_AL, [np.zeros(3)]),
    ("Tl.pbe-d-hgh.upf", FCC_AL, [np.zeros(3)])])
def test_basis_form_factors_match_oracle(name, lattice, positions):
    """P, the local potential and ρcore of a UPF basis at 1e-12 relative."""
    from oracle.basis import PlaneWaveBasis as OBasis
    from oracle.terms import Terms, build_projection_vectors
    from oracle.nlcc import core_density
    dftk, pm, om = _models(name, lattice, positions, ("lda_x", "lda_c_pw"), symmetries=False)
    kc = [[0.1, 0.2, -0.3], [0.0, 0.0, 0.0]]
    basis = dftk.PlaneWaveBasis(pm, Ecut=12, kgrid=dftk.ExplicitKpoints(kc, [0.5, 0.5]))
    ob = OBasis(om, 12, fft_size=basis.fft_size, kcoords=kc, kweights=[0.5, 0.5])
    vloc = basis.term("AtomicLocal").potential_values.cpu().numpy()
    oref = Terms(ob).Vloc
    assert np.abs(vloc - oref).max() <= 1e-12 * np.abs(oref).max()
    for ik, kpt in enumerate(basis.kpoints):
        P = basis.term("AtomicNonlocal").ops[ik].P.cpu().numpy().T
        Pref, Dref = build_projection_vectors(ob, ob.kpoints[ik])
        assert P.shape == Pref.shape
        assert np.abs(P - Pref).max() <= 1e-12 * np.abs(Pref).max()
        np.testing.assert_array_equal(basis.term("AtomicNonlocal").ops[ik].D, Dref)
    rc = basis.term("Xc").rho_core
    orc = core_density(ob)
    if orc is None:
        assert rc is None
    else:
        assert np.abs(rc.cpu().numpy() - orc).max() <= 1e-12 * np.abs(orc).max()


def _scf_pair(dftk, pm, om, Ecut, kgrid, tol=1e-9, **okw):
    from oracle.basis import PlaneWaveBasis as OBasis
    from oracle import nlcc
    basis = dftk.PlaneWaveBasis(pm, Ecut=Ecut, kgrid=kgrid)
    res = dftk.self_consistent_field(basis, tol=tol)
    assert res["converged"]
    ob = OBasis(om, Ecut, kgrid=kgrid)
    assert ob.fft_size == basis.fft_size and len(ob.kpoints) == len(basis.kpoints)
    ores = nlcc.self_consistent_field(ob, tol=tol, **okw)
    assert ores["converged"]
    return basis, res, ob, ores


def _compare(basis, res, ob, ores, n_atoms, n_eig):
    """BASELINE tolerances: energy 1e-8 Ha/atom, eigenvalues 1e-6 Ha, density L2 1e-7."""
    assert abs(res["energies"].total - ores["energies"]["total"]) < 1e-8 * n_atoms
    for ik, kpt in enumerate(basis.kpoints):
        jk = [j for j, ok in enumerate(ob.kpoints) if np.allclose(ok.coordinate, kpt.coordinate) and ok.spin == kpt.spin][0]
        np.testing.assert_allclose(res["eigenvalues"][ik][:n_eig], ores["eigenvalues"][jk][:n_eig], atol=1e-6)
    drho = res["rho"].cpu().numpy() - ores["rho"]
    assert np.linalg.norm(drho) * math.sqrt(basis.dvol) < 1e-7


def test_scf_carbon_lda_nlcc_matches_oracle():
    dftk, pm, om = _models("C_m.upf", DIAMOND, [np.ones(3) / 8, -np.ones(3) / 8], dftk_lda())
    basis, res, ob, ores = _scf_pair(dftk, pm, om, 10, (2, 2, 2))
    assert basis.term("Xc").rho_core is not None
    _compare(basis, res, ob, ores, 2, 4)


def test_scf_aluminium_pbe_smearing_nlcc_matches_oracle():
    dftk, pm, om = _models("Al_m.upf", FCC_AL, [np.zeros(3)], ("gga_x_pbe", "gga_c_pbe"), temperature=0.01)
    basis, res, ob, ores = _scf_pair(dftk, pm, om, 10, (3, 3, 3))
    _compare(basis, res, ob, ores, 1, 2)


def test_scf_collinear_spin_nlcc_matches_oracle():
    dftk, pm, om = _models("C_m.upf", DIAMOND, [np.ones(3) / 8, -np.ones(3) / 8], dftk_lda(), magnetic_moments=[1.0, 1.0],
                           temperature=0.01)
    basis, res, ob, ores = _scf_pair(dftk, pm, om, 10, (1, 1, 1))
    assert pm.n_spin_components == 2
    rc = basis.term("Xc").rho_core
    torch.testing.assert_close(rc[0], rc[1], rtol=0, atol=0)
    _compare(basis, res, ob, ores, 2, 4)


def dftk_lda():
    return ("lda_x", "lda_c_pw")


def test_silicon_pbe_upf_matches_analytic_hgh():
    """Si.pbe-hgh.upf is the numerical form of the analytic GTH-PBE-q4 pseudopotential.  On the CPU oracle the two SCF
    total energies of this setup (Ecut 10, 2×2×2 k-grid) differ by 4.1e-8 Ha; the bound allows 2e-7."""
    import dftk_b200 as dftk
    up = dftk.ElementPsp("Si", psp=product_psp("Si.pbe-hgh.upf"))
    an = dftk.ElementPsp("Si", psp=dftk.load_psp(os.path.join(UPF, "Si-q4.gth")))
    E = []
    for el in (up, an):
        model = dftk.model_DFT(LATTICE, [el, el], POSITIONS, functionals=dftk.PBE())
        basis = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=(2, 2, 2))
        res = dftk.self_consistent_field(basis, tol=1e-9)
        assert res["converged"]
        E.append(res["energies"].total)
    assert abs(E[0] - E[1]) < 2e-7


def test_nlcc_forces_match_oracle():
    """Same ψ, occupation and ρ on both sides (the oracle's SCF of a displaced C₂ cell): every term, the NLCC one on
    its own, to 1e-10."""
    from oracle.basis import PlaneWaveBasis as OBasis
    from oracle import nlcc
    pos = [np.ones(3) / 8 + np.array([0.012, -0.006, 0.004]), -np.ones(3) / 8]
    dftk, pm, om = _models("C_m.upf", DIAMOND, pos, dftk_lda(), symmetries=False)
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
