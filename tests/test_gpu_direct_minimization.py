"""direct_minimization on the device: against the SCF (reference: test/scf_compare.jl), the gradient against finite
differences of the energy, the first iterations against the NumPy twin on the oracle, bit-for-bit reproducibility, the
large-block path, launch counts independent of the block count, forces of its result, and its refusals."""
import math
import numpy as np
import pytest
import torch

import dftk_b200 as dftk
from dftk_b200 import device as dev
from dftk_b200.direct_minimization import energy_gradient, stiefel_retract, DeviceOps
from silicon import LATTICE, POSITIONS, KCOORDS, KWEIGHTS

pytestmark = pytest.mark.gpu


def _si_model(positions=POSITIONS, lattice=LATTICE, n_atoms=2, **kw):
    Si = dftk.ElementPsp("Si", functional="lda")
    return dftk.model_DFT(lattice, [Si] * n_atoms, positions, functionals=["lda_x", "lda_c_vwn"], **kw)


def _ref_basis(**kw):
    return dftk.PlaneWaveBasis(_si_model(**kw), Ecut=3, kgrid=dftk.ExplicitKpoints(KCOORDS, KWEIGHTS), fft_size=(9, 9, 9))


def _linf(a, b):
    return float((a - b).abs().max())


def test_dm_matches_scf_spinless():
    tol = 1e-7
    basis = _ref_basis()
    ref = dftk.self_consistent_field(basis, tol=tol / 10)
    res = dftk.direct_minimization(basis, tol=tol)
    assert res["algorithm"] == "DM" and res["stage"] == "finalize" and res["eF"] is None
    assert _linf(res["rho"], ref["rho"]) < 10 * tol
    assert abs(res["energies"].total - ref["energies"].total) < 1e-8
    # the final Rayleigh-Ritz gives the occupied eigenvalues of the SCF
    for ek, rk in zip(res["eigenvalues"], ref["eigenvalues"]):
        np.testing.assert_allclose(ek, rk[:4], atol=1e-6)
    for p in res["psi"]:
        G = (p.conj() @ p.T).cpu().numpy()
        np.testing.assert_allclose(G, np.eye(4), atol=1e-12)


def test_dm_matches_scf_collinear():
    tol = 1e-7
    mm = [1.0, 1.0]
    basis = _ref_basis(magnetic_moments=mm)
    rho0 = dftk.guess_density(basis, mm)
    ref = dftk.self_consistent_field(basis, rho=rho0, tol=tol / 10)
    start = dftk.self_consistent_field(basis, rho=rho0, tol=tol, maxiter=1)
    psi = dftk.select_occupied_orbitals(basis, start["psi"], start["occupation"])["psi"]
    res = dftk.direct_minimization(basis, psi=psi, tol=tol)
    assert _linf(res["rho"], ref["rho"]) < 10 * tol
    assert abs(res["energies"].total - ref["energies"].total) < 1e-8


def test_energy_convergence_criterion():
    basis = _ref_basis()
    ref = dftk.self_consistent_field(basis, tol=1e-8)
    seen = []
    res = dftk.direct_minimization(basis, is_converged=dftk.ScfConvergenceEnergy(1e-10),
                                   callback=lambda info: seen.append((info["rho"], info["rho_in"])))
    assert res["converged"]
    h = res["history_Etot"]
    assert abs(h[-1] - h[-2]) < 1e-10
    assert abs(res["energies"].total - ref["energies"].total) < 1e-8
    # the callback sees the reference's keys: rho is the density of the next step's orbitals, rho_in the current one
    rho_out, rho_in = seen[-1]
    assert res["history_drho"][-1] == pytest.approx(float((rho_out - rho_in).norm()) * math.sqrt(basis.dvol), rel=1e-14)


def _tangent(basis, psi, seed):
    g = torch.Generator(device=psi[0].device).manual_seed(seed)
    D = [torch.randn(p.shape, dtype=torch.complex128, device=p.device, generator=g) for p in psi]
    dev.stiefel_project_multi(basis.kblocks, psi, D)
    nrm = math.sqrt(dev.real_dots_multi(basis.kblocks, [(D, D)])[0])
    return [d / nrm for d in D]


@pytest.mark.parametrize("collinear", [False, True])
def test_gradient_is_the_energy_derivative(collinear):
    kw = dict(magnetic_moments=[1.0, 1.0]) if collinear else {}
    basis = dftk.PlaneWaveBasis(_si_model(**kw), Ecut=6, kgrid=(2, 2, 2))
    assert len(basis.model.symmetries) > 1 and len(basis.kpoints) > 1
    nb = 4
    psi = dev.random_orbitals_multi(basis.kblocks, nb, 11)
    E0, G = energy_gradient(basis, psi)
    D = _tangent(basis, psi, 5)
    pred = dev.real_dots_multi(basis.kblocks, [(G, D)])[0]
    def E(t):
        return energy_gradient(basis, stiefel_retract(basis, [p + t * d for p, d in zip(psi, D)]))[0]

    def central(h):
        return (E(h) - E(-h)) / (2 * h)
    fd = (4 * central(5e-4) - central(1e-3)) / 3          # Richardson: O(h^4)
    assert abs(pred) > 1e-3
    assert abs(fd - pred) < 1e-6 * abs(pred)


def test_retraction_is_the_polar_factor_and_projection_is_tangent():
    basis = dftk.PlaneWaveBasis(_si_model(), Ecut=6, kgrid=(2, 2, 2))
    psi = dev.random_orbitals_multi(basis.kblocks, 4, 3)
    g = torch.Generator(device=psi[0].device).manual_seed(1)
    Y = [p + 0.3 * torch.randn(p.shape, dtype=torch.complex128, device=p.device, generator=g) for p in psi]
    X = stiefel_retract(basis, Y)
    for y, x in zip(Y, X):
        yn, xn = y.cpu().numpy().T, x.cpu().numpy().T
        U, _, Vh = np.linalg.svd(yn, full_matrices=False)
        np.testing.assert_allclose(xn, U @ Vh, atol=1e-12)
    D = _tangent(basis, X, 2)
    for x, d in zip(X, D):
        C = (x.conj() @ d.T).cpu().numpy()                   # X^H D must be anti-Hermitian
        np.testing.assert_allclose(C + C.conj().T, 0, atol=1e-12)


@pytest.mark.parametrize("prec_type", ["TPA", None])
def test_first_iterations_match_the_oracle(prec_type):
    import dm_oracle
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    basis = _ref_basis(symmetries=False)
    om = Model(LATTICE, [Element("Si")] * 2, POSITIONS, functionals=("lda_x", "lda_c_vwn"), symmetries=False)
    ob = OBasis(om, 3, fft_size=(9, 9, 9), kcoords=KCOORDS, kweights=KWEIGHTS)
    for k, ok in zip(basis.kpoints, ob.kpoints):
        assert np.array_equal(k.mapping.cpu().numpy(), ok.mapping)
    psi = dev.random_orbitals_multi(basis.kblocks, 4, 77)
    never = lambda info: False
    res = dftk.direct_minimization(basis, psi=[p.clone() for p in psi], maxiter=6, is_converged=never, prec_type=prec_type)
    ores = dm_oracle.direct_minimization(ob, [p.cpu().numpy().T.copy() for p in psi], maxiter=6, is_converged=never,
                                         prec_type=prec_type)
    np.testing.assert_allclose(res["history_Etot"][:5], ores["history_Etot"][:5], rtol=1e-10)


def test_runs_are_bit_identical():
    basis = dftk.PlaneWaveBasis(_si_model(), Ecut=6, kgrid=(3, 3, 3))
    psi = dev.random_orbitals_multi(basis.kblocks, 4, 9)
    never = lambda info: False
    h = [dftk.direct_minimization(basis, psi=[p.clone() for p in psi], maxiter=8, is_converged=never)["history_Etot"]
         for _ in range(2)]
    assert h[0] == h[1]


def test_large_blocks_at_gamma():
    rep = (2, 2, 3)
    lat = LATTICE * np.array(rep)[None, :]
    pos = [(np.asarray(p) + np.array([i, j, k])) / np.array(rep) for i in range(rep[0]) for j in range(rep[1])
           for k in range(rep[2]) for p in POSITIONS]
    model = _si_model(positions=pos, lattice=lat, n_atoms=len(pos), symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=4, kgrid=(1, 1, 1))
    assert basis.kblocks[0].fold_size() > 0
    tol = 1e-6
    ref = dftk.self_consistent_field(basis, tol=tol / 10)
    res = dftk.direct_minimization(basis, tol=tol, seed=1)
    assert res["psi"][0].shape[0] == 48
    assert _linf(res["rho"], ref["rho"]) < 10 * tol
    assert abs(res["energies"].total - ref["energies"].total) < 1e-8


def _iteration_launches(n_k):
    rng = np.random.default_rng(n_k)
    kc = [list(rng.uniform(-0.5, 0.5, 3)) for _ in range(n_k)]
    basis = dftk.PlaneWaveBasis(_si_model(symmetries=False), Ecut=7, kgrid=dftk.ExplicitKpoints(kc),
                                fft_size=(18, 18, 18))
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=dftk.guess_density(basis))
    kbs = [ham[ik].bind() for ik in range(n_k)]
    ops = DeviceOps(basis, 4, "TPA")
    x = dev.random_orbitals_multi(basis.kblocks, 4, 1)
    g = dev.random_orbitals_multi(basis.kblocks, 4, 2)
    ctx = basis.architecture.ctx
    ctx.sync()
    ctx.launch_count(reset=True)
    # the device operations of one iteration with one history pair: gradient, projections, preconditioner, two-loop dots
    # and fused updates, one line-search point
    dev.apply_h_multi(kbs, x, g, scale=[2.0 * w for w in basis.kweights])
    ops.project(x, g)
    ops.precondprep(x)
    q = ops.copy(g)
    d = ops.dot(x, q)
    d = ops.axpy_dot(q, g, -0.1, x)
    s = ops.ldiv(q)
    d = ops.axpy_dot(s, x, 0.2, None)
    ops.negate(s)
    ops.project(x, s)
    y = ops.retract(ops.add_scaled(x, s, 0.5))
    ctx.sync()
    return ctx.launch_count()


def test_launch_count_does_not_depend_on_the_block_count():
    assert _iteration_launches(4) == _iteration_launches(16)


def test_forces_of_the_dm_result():
    pos = [POSITIONS[0] + np.array([0.01, -0.005, 0.0]), POSITIONS[1]]
    basis = dftk.PlaneWaveBasis(_si_model(positions=pos, symmetries=False), Ecut=6, kgrid=(2, 2, 2))
    scf = dftk.self_consistent_field(basis, tol=1e-10)
    res = dftk.direct_minimization(basis, tol=1e-9)
    f_scf = np.array(dftk.compute_forces(scf))
    f_dm = np.array(dftk.compute_forces(res))
    assert np.abs(f_scf).max() > 1e-3
    np.testing.assert_allclose(f_dm, f_scf, atol=1e-6)


def test_refusals():
    basis = dftk.PlaneWaveBasis(_si_model(temperature=0.01), Ecut=3, kgrid=(1, 1, 1), fft_size=(9, 9, 9))
    with pytest.raises(ValueError):
        dftk.direct_minimization(basis)
    from upf_data import product_psp
    Si = dftk.ElementPsp("Si", product_psp("Si.pbe-hgh.upf"))
    model = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(),
                           extra_terms=[dftk.Hubbard((dftk.OrbitalManifold("Si", "3P"), 0.1))])
    basis = dftk.PlaneWaveBasis(model, Ecut=6, kgrid=(1, 1, 1))
    with pytest.raises(NotImplementedError):
        dftk.direct_minimization(basis)
    basis = _ref_basis()
    with pytest.raises(ValueError):
        dftk.direct_minimization(basis, psi=[torch.zeros((5, k.n_G), dtype=torch.complex128) for k in basis.kpoints])
