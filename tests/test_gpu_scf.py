"""End-to-end GPU parity: the product's Model / PlaneWaveBasis / self_consistent_field path (all orbital
work inside libdftk_b200) against (a) the reference's own golden numbers and (b) the CPU oracle."""
import math
import os
import numpy as np
import pytest
import torch

from silicon import LATTICE, POSITIONS, KCOORDS, KWEIGHTS

pytestmark = pytest.mark.gpu


def _si_model(dftk, functionals, **kw):
    Si = dftk.ElementPsp("Si", functional="lda")
    return dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=functionals, **kw)


def test_energies_guess_density_golden():
    # reference: test/energies_guess_density.jl:8-36 -- every energy term pinned to 5e-8
    import dftk_b200 as dftk
    model = _si_model(dftk, ["lda_x", "lda_c_vwn"], symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=15, kgrid=dftk.MonkhorstPack((1, 2, 3), kshift=(0, 0.5, 0)),
                                fft_size=(27, 27, 27))
    rho0 = dftk.guess_density(basis)
    E, ham = dftk.energy_hamiltonian(basis, None, None, rho=rho0)
    assert E["Hartree"] == pytest.approx(0.3527293727197568, abs=5e-8)
    assert E["Xc"] == pytest.approx(-2.3033165870558165, abs=5e-8)
    res = dftk.diagonalize_all_kblocks(dftk.lobpcg_hyper, ham, 8, tol=1e-9)
    assert all(np.max(r[:4]) < 1e-8 for r in res["residual_norms"])
    occ = [np.array([2., 2, 2, 2, 0, 0, 0, 0]) for _ in basis.kpoints]
    rho = dftk.compute_density(basis, res["X"], occ)
    E, _ = dftk.energy_hamiltonian(basis, res["X"], occ, rho=rho)
    ref = dict(Kinetic=3.3824289861522194, AtomicLocal=-2.4178712046759157, AtomicNonlocal=1.664289455206788,
               Hartree=0.6712993199211524, Xc=-2.4489960475309056, Ewald=-8.397893578467201,
               PspCorrection=-0.294622067031369)
    for k, v in ref.items():
        assert E[k] == pytest.approx(v, abs=5e-8), k


def test_scf_matches_oracle_with_symmetries():
    # BASELINE tolerances: energy 1e-8 Ha/atom, eigenvalues 1e-6 Ha, density L2 1e-7
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle import scf as oscf
    model = _si_model(dftk, dftk.LDA())
    assert len(model.symmetries) == 48
    basis = dftk.PlaneWaveBasis(model, Ecut=12, kgrid=(3, 3, 3))
    res = dftk.self_consistent_field(basis, tol=1e-9)
    assert res["converged"]
    om = Model(LATTICE, [Element("Si")] * 2, POSITIONS, functionals=("lda_x", "lda_c_pw"))
    ob = OBasis(om, 12, kgrid=(3, 3, 3))
    assert ob.fft_size == basis.fft_size
    assert len(ob.kpoints) == len(basis.kpoints)
    ores = oscf.self_consistent_field(ob, tol=1e-9)
    assert abs(res["energies"].total - ores["energies"]["total"]) < 2e-8          # 1e-8 Ha/atom, 2 atoms
    for name in ("Kinetic", "AtomicLocal", "AtomicNonlocal", "Hartree", "Xc", "Ewald", "PspCorrection"):
        assert abs(res["energies"][name] - ores["energies"][name]) < 1e-7, name
    # k-point order may differ between the two orbit searches: match by coordinate
    for ik, kpt in enumerate(basis.kpoints):
        jk = [j for j, ok in enumerate(ob.kpoints) if np.allclose(ok.coordinate, kpt.coordinate)][0]
        assert abs(basis.kweights[ik] - ob.kweights[jk]) < 1e-14
        np.testing.assert_allclose(res["eigenvalues"][ik][:4], ores["eigenvalues"][jk][:4], atol=1e-6)
    drho = res["rho"].cpu().numpy() - ores["rho"]
    assert np.linalg.norm(drho) * math.sqrt(basis.dvol) < 1e-7


def test_silicon_lda_vs_abinit():
    # reference: test/silicon_lda.jl:10-20,47-51 (Ecut 25, fft 33³; eigenvalues and Etot to 1e-5)
    import dftk_b200 as dftk
    model = _si_model(dftk, ["lda_x", "lda_c_vwn"])
    basis = dftk.PlaneWaveBasis(model, Ecut=25, kgrid=dftk.ExplicitKpoints(KCOORDS, KWEIGHTS), fft_size=(33, 33, 33))
    ref = [[-0.178566465714968, 0.261882541175914, 0.261882541178847, 0.261882541181782,
            0.354070367072414, 0.354070367076363, 0.354070367080310, 0.376871160884678],
           [-0.127794342370963, 0.064395861472044, 0.224958824747686, 0.224958824750934,
            0.321313617512188, 0.388442495007398, 0.388442495010722, 0.542078732298094],
           [-0.108449612789883, 0.077125812982728, 0.172380374761464, 0.172380374766260,
            0.283802499666810, 0.329872296009131, 0.525606867582028, 0.525606867585921],
           [-0.058089253154566, 0.012364292440522, 0.097350168867990, 0.183765652148129,
            0.314593174568090, 0.470869435132365, 0.496966579772700, 0.517009645871194]]
    res = dftk.self_consistent_field(basis, is_converged=dftk.ScfConvergenceEnergy(1e-7),
                                     nbandsalg=dftk.AdaptiveBands(model, n_bands_converge=8))
    assert res["energies"].total == pytest.approx(-7.911817522631488, abs=1e-5)
    for ik in range(4):
        np.testing.assert_allclose(res["eigenvalues"][ik][:8], ref[ik], atol=1e-5)


def test_silicon_pbe_vs_abinit():
    # reference: test/silicon_pbe.jl:6-41,57-61 (Ecut 25, fft 33; eigenvalues and E_tot to 1e-5)
    import dftk_b200 as dftk
    Si = dftk.ElementPsp("Si", functional="pbe")
    model = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.PBE())
    basis = dftk.PlaneWaveBasis(model, Ecut=25, kgrid=dftk.ExplicitKpoints(KCOORDS, KWEIGHTS), fft_size=(33, 33, 33))
    ref = [[-0.181210259413818, 0.258840553222639, 0.258840553225549, 0.258840553228459, 0.351692348652324,
            0.351692348656259, 0.351692348660193, 0.380606400669216, 0.540705881744348, 0.540705883460555],
           [-0.130553299114991, 0.062256443775155, 0.221871391287580, 0.221871391290802, 0.322398722411882,
            0.386194327436667, 0.386194327439986, 0.546859898649217, 0.550571701390781, 0.550571701394327],
           [-0.111170738096744, 0.074494899973125, 0.169461730083372, 0.169461730088140, 0.284305392082236,
            0.330468937070505, 0.524509288492752, 0.524509288496625, 0.616964090764029, 0.619623658242765],
           [-0.061054203629684, 0.009700769243041, 0.095769985640881, 0.180784778430457, 0.315000287382235,
            0.471042322838057, 0.495281775946584, 0.517469860611792, 0.530124341745161, 0.539044739392045]]
    res = dftk.self_consistent_field(basis, is_converged=dftk.ScfConvergenceEnergy(1e-8),
                                     nbandsalg=dftk.AdaptiveBands(model, n_bands_converge=10))
    assert res["energies"].total == pytest.approx(-7.854477356672080, abs=1e-5)
    for ik in range(4):
        np.testing.assert_allclose(res["eigenvalues"][ik][:10], ref[ik], atol=1e-5)


def test_iron_pbe_collinear_vs_abinit():
    # reference: test/iron_pbe.jl:6-70 (GTH-PADE-q8, PBE, collinear spin, T = 0.01, Ecut 20, fft 20, shifted 4x4x4 grid)
    import dftk_b200 as dftk
    fe_q8 = ("Fe GTH-PADE-q8 GTH-LDA-q8\n    2    0    6\n     0.61000000    0\n    3\n"
             "     0.45448200    3     3.01664046    -1.00040646     0.79478164\n"
             "                                        2.58303836    -2.05211737\n"
             "                                                       3.25763534\n"
             "     0.63890282    2     1.49964199    -0.13812935\n"
             "                                        0.32687369\n"
             "     0.30873177    1    -9.14535371\n")
    Fe = dftk.ElementPsp("Fe", psp=dftk.parse_hgh(fe_q8, identifier="hgh/lda/fe-q8"))
    assert Fe.psp.Zion == 8 and Fe.psp.count_n_proj() == 14
    lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
    model = dftk.model_DFT(lat, [Fe], [[0, 0, 0]], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0])
    basis = dftk.PlaneWaveBasis(model, Ecut=20, kgrid=dftk.MonkhorstPack((4, 4, 4), kshift=(0.5, 0.5, 0.5)), fft_size=(20, 20, 20))
    assert len(basis.kpoints) == 12
    res = dftk.self_consistent_field(basis, rho=dftk.guess_density(basis, [4.0]), mixing=dftk.KerkerMixing(),
                                     is_converged=dftk.ScfConvergenceEnergy(1e-10),
                                     nbandsalg=dftk.AdaptiveBands(model, n_bands_converge=10))
    assert res["energies"].total == pytest.approx(-18.21465922614397, abs=5e-6)
    mag = float((res["rho"][0] - res["rho"][1]).sum() * basis.dvol)
    assert mag == pytest.approx(2.98199463, abs=5e-5)
    # spot values of the ABINIT spectra (first and last irreducible k-point of each spin channel are matched by value)
    lowest = sorted(float(e[0]) for e in res["eigenvalues"])
    ref_lowest = sorted([0.0603597727989307, 0.1384929268069029, -0.017996603976028, 0.1102557166995405, 0.1723514110126840,
                         0.1360541296075938, 0.0802990962833626, 0.2341496631160049, -0.002234753604747, 0.1518900787487526,
                         0.2873355363445261, 0.2512356397409882])
    np.testing.assert_allclose(lowest, ref_lowest, atol=5e-6)


def test_hamiltonian_consistency():
    # reference: test/hamiltonian_consistency.jl:54-58 -- operator application equals the dense matrix
    import dftk_b200 as dftk
    model = _si_model(dftk, dftk.LDA(), symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=3, kgrid=dftk.ExplicitKpoints([[0.2, 0.3, 0.1]]), fft_size=(15, 15, 15))
    rho = dftk.guess_density(basis)
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=rho)
    blk = ham[0]
    n = blk.kpoint.n_G
    I = torch.eye(n, dtype=torch.complex128, device=rho.device)
    H = blk.mul(I).T          # column j = H e_j  -> dense matrix (n x n)
    assert (H - H.conj().T).abs().max().item() < 1e-10       # Hermitian
    psi = dftk.random_orbitals(basis, blk.kpoint, 5)
    np.testing.assert_allclose(blk.mul(psi).cpu().numpy(), (psi @ H.T).cpu().numpy(), atol=1e-11)
    w = torch.linalg.eigvalsh(H)[:4].cpu().numpy()
    res = dftk.diagonalize_all_kblocks(dftk.lobpcg_hyper, ham, 4, tol=1e-9)
    np.testing.assert_allclose(res["λ"][0], w, atol=1e-8)       # "Full diagonalization" check, test/lobpcg.jl:105+


def _compare_scf(res, ores, basis, ob, n_atoms, n_cmp):
    assert abs(res["energies"].total - ores["energies"]["total"]) < 1e-8 * max(1, n_atoms) + 1e-9
    for ik, kpt in enumerate(basis.kpoints):
        jk = [j for j, ok in enumerate(ob.kpoints) if ok.spin == kpt.spin and np.allclose(ok.coordinate, kpt.coordinate)][0]
        np.testing.assert_allclose(res["eigenvalues"][ik][:n_cmp], ores["eigenvalues"][jk][:n_cmp], atol=1e-6)
    drho = res["rho"].cpu().numpy() - ores["rho"]
    assert np.linalg.norm(drho) * math.sqrt(basis.dvol) < 1e-7


def test_aluminium_pbe_smearing_matches_oracle():
    # BASELINE config C4 shape (Al fcc 4-atom PBE, Fermi-Dirac smearing, Kerker mixing), reduced Ecut / k-grid
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle import scf as oscf
    a = 7.65339
    lat = a * np.eye(3)
    pos = [[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]]
    Al = dftk.ElementPsp("Al", functional="pbe")
    model = dftk.model_DFT(lat, [Al] * 4, pos, functionals=dftk.PBE(), temperature=0.01)
    assert len(model.symmetries) == 192
    basis = dftk.PlaneWaveBasis(model, Ecut=7, kgrid=(2, 2, 2))
    res = dftk.self_consistent_field(basis, tol=1e-9, mixing=dftk.KerkerMixing())
    assert res["converged"]
    om = Model(lat, [Element("Al", functional="pbe")] * 4, pos, functionals=("gga_x_pbe", "gga_c_pbe"), temperature=0.01)
    ob = OBasis(om, 7, kgrid=(2, 2, 2))
    assert ob.fft_size == basis.fft_size and len(ob.kpoints) == len(basis.kpoints)
    ores = oscf.self_consistent_field(ob, tol=1e-9, mixing="kerker")
    assert abs(res["eF"] - ores["eF"]) < 1e-6
    assert abs(res["energies"]["Entropy"] - ores["energies"]["Entropy"]) < 1e-7
    _compare_scf(res, ores, basis, ob, 4, 6)


def test_aluminium_default_ldos_mixing_matches_oracle():
    """The reference's DEFAULT mixing (LdosMixing, self_consistent_field.jl:177; mixing.jl:205-292): product default vs the
    oracle's restatement (same chi0 model, same GMRES): energy, Fermi level and the number of SCF iterations."""
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle import scf as oscf
    a = 7.65339
    pos = [[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]]
    Al = dftk.ElementPsp("Al", functional="pbe")
    model = dftk.model_DFT(a * np.eye(3), [Al] * 4, pos, functionals=dftk.PBE(), temperature=0.01)
    basis = dftk.PlaneWaveBasis(model, Ecut=7, kgrid=(2, 2, 2))
    res = dftk.self_consistent_field(basis, tol=1e-9)                        # mixing = LdosMixing() by default
    assert res["converged"]
    om = Model(a * np.eye(3), [Element("Al", functional="pbe")] * 4, pos, functionals=("gga_x_pbe", "gga_c_pbe"), temperature=0.01)
    ob = OBasis(om, 7, kgrid=(2, 2, 2))
    ores = oscf.self_consistent_field(ob, tol=1e-9, mixing="ldos")
    assert abs(res["energies"].total - ores["energies"]["total"]) < 4e-8     # 1e-8 Ha/atom
    assert abs(res["eF"] - ores["eF"]) < 1e-6
    assert abs(res["n_iter"] - ores["n_iter"]) <= 2
    # the LDOS itself: one more density pass with -f' weights (dos.jl:43-65) vs the oracle's
    ld = dftk.compute_ldos(basis, res["eF"], res["eigenvalues"], res["psi"], temperature=0.1)
    old = oscf.compute_ldos(ob, ores["eF"], ores["eigenvalues"], ores["psi"], 0.1)
    assert np.linalg.norm(ld.cpu().numpy() - old) * math.sqrt(basis.dvol) < 1e-6 * np.linalg.norm(old) * math.sqrt(basis.dvol) + 1e-7


def test_mixing_helpers_on_device():
    """dftk_b200_tall_gram (Anderson / GMRES history dot products in one launch) and the device Anderson against NumPy."""
    import dftk_b200 as dftk
    from gpu_common import ctx
    c = ctx()
    g = torch.Generator(device="cpu").manual_seed(0)
    A = torch.randn(5, 20000, generator=g, dtype=torch.float64).to(c.device)
    B = torch.randn(3, 20000, generator=g, dtype=torch.float64).to(c.device)
    np.testing.assert_allclose(c.real_gram(A, B), (A @ B.T).cpu().numpy(), rtol=1e-12, atol=1e-10)
    # Anderson on the device reproduces the host path on a linear fixed-point problem (test/anderson.jl)
    n = 401                                                                    # odd length: exercises the padding
    M = torch.randn(n, n, generator=g, dtype=torch.float64) * (0.3 / math.sqrt(n))
    b = torch.randn(n, generator=g, dtype=torch.float64)
    xs = {}
    for dev in ("cpu", "cuda"):
        Md, bd = M.to(dev), b.to(dev)
        acc = dftk.AndersonAcceleration(m=10, ctx=c if dev == "cuda" else None)
        x = torch.zeros(n, dtype=torch.float64, device=dev)
        for _ in range(12):
            x = acc(x, 0.8, Md @ x + bd - x)
        xs[dev] = x.cpu()
    xstar = torch.linalg.solve(torch.eye(n, dtype=torch.float64) - M, b)
    assert (xs["cuda"] - xstar).abs().max().item() < 1e-4          # 12 steps with a history of 10 on a 401-dimensional problem
    assert (xs["cuda"] - xs["cpu"]).abs().max().item() < 1e-9      # Gram + refinement on the device == QR-free host path


def test_random_orbitals_are_orthonormal():
    import dftk_b200 as dftk
    model = _si_model(dftk, dftk.LDA(), symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=8, kgrid=dftk.ExplicitKpoints([[0.2, 0.3, 0.1], [0, 0, 0]], [0.5, 0.5]), fft_size=(18, 18, 18))
    from dftk_b200.device import random_orbitals_multi
    Xs = random_orbitals_multi(basis.kblocks, 9, seed=5)
    for X in Xs:
        G = X.conj() @ X.T
        assert (G - torch.eye(9, dtype=G.dtype, device=G.device)).abs().max().item() < 1e-13
    assert (Xs[0][:, :50] - Xs[1][:, :50]).abs().max().item() > 1e-3            # different blocks, different numbers
    Y = random_orbitals_multi(basis.kblocks, 9, seed=5)
    assert torch.equal(Y[0], Xs[0])                                              # deterministic in the seed


def test_iron_collinear_spin_matches_oracle():
    # BASELINE config C5 shape (Fe bcc PBE, collinear spin), reduced Ecut / k-grid; test/iron_pbe.jl:53 setup
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle import scf as oscf
    lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
    Fe = dftk.ElementPsp("Fe", functional="pbe")
    model = dftk.model_DFT(lat, [Fe], [[0, 0, 0]], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0])
    assert model.n_spin_components == 2
    basis = dftk.PlaneWaveBasis(model, Ecut=20, kgrid=(3, 3, 3))
    res = dftk.self_consistent_field(basis, tol=1e-8, mixing=dftk.KerkerMixing())
    assert res["converged"]
    om = Model(lat, [Element("Fe", functional="pbe")], [[0, 0, 0]], functionals=("gga_x_pbe", "gga_c_pbe"),
               temperature=0.01, magnetic_moments=[4.0])
    ob = OBasis(om, 20, kgrid=(3, 3, 3))
    assert ob.fft_size == basis.fft_size and len(ob.kpoints) == len(basis.kpoints)
    ores = oscf.self_consistent_field(ob, tol=1e-8, mixing="kerker")
    mag = float((res["rho"][0] - res["rho"][1]).sum() * basis.dvol)
    omag = float((ores["rho"][0] - ores["rho"][1]).sum() * ob.dvol)
    assert abs(mag - omag) < 1e-5 and mag > 0.5
    assert abs(res["energies"].total - ores["energies"]["total"]) < 1e-7      # reference GPU test: 1e-7 for Fe (test/gpu.jl:72)
    for ik, kpt in enumerate(basis.kpoints):
        jk = [j for j, ok in enumerate(ob.kpoints) if ok.spin == kpt.spin and np.allclose(ok.coordinate, kpt.coordinate)][0]
        np.testing.assert_allclose(res["eigenvalues"][ik][:8], ores["eigenvalues"][jk][:8], atol=1e-6)
    assert np.linalg.norm(res["rho"].cpu().numpy() - ores["rho"]) * math.sqrt(basis.dvol) < 1e-6   # test/gpu.jl:73


@pytest.mark.parametrize("rep,Ecut,fft", [(2, 8, 18), (3, 12, 24)])
def test_supercell_identity(rep, Ecut, fft):
    # reference: test/supercell.jl:19-45 -- a Gamma-only rep^3 supercell equals the unit cell with a rep^3 k-grid
    # (E_super = rep^3 E_unit to 1e-8 Ha per unit cell; supercell fft = unit fft x rep, supercell.jl:35).  This is the cheap
    # oracle of the C3 cell (Gamma-only supercell <-> k-grid of the primitive cell): rep = 2 runs 35 bands, rep = 3 runs
    # 54 atoms / 111 bands on a 72^3 grid through the large LOBPCG path (tensor-core GEMMs, cuSOLVER, locking).
    import dftk_b200 as dftk
    Si = dftk.ElementPsp("Si")
    n = rep ** 3
    unit = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), symmetries=False)
    bu = dftk.PlaneWaveBasis(unit, Ecut=Ecut, kgrid=(rep, rep, rep), fft_size=(fft, fft, fft))
    ru = dftk.self_consistent_field(bu, tol=1e-9)
    pos = [(np.asarray(p) + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep) for p in POSITIONS]
    sup = dftk.model_DFT(rep * LATTICE, [Si] * (2 * n), pos, functionals=dftk.LDA(), symmetries=False)
    bs = dftk.PlaneWaveBasis(sup, Ecut=Ecut, kgrid=(1, 1, 1), fft_size=(rep * fft,) * 3)
    rs = dftk.self_consistent_field(bs, tol=1e-9)
    assert rs["converged"] and ru["converged"]
    assert abs(rs["energies"].total - n * ru["energies"].total) < n * 1e-8
    assert abs(float(rs["rho"].sum() * bs.dvol) - 8.0 * n) < 1e-9


def test_supercell_identity_on_int8_tensor_cores():
    """The same identity (rep = 3: 54 atoms, 111 bands, 72^3 grid) with the Gram products of LOBPCG and the P'psi projection
    on the INT8 tensor cores (gemm_backend 4: FP64 emulated by INT8 residues + CRT, wgmma s8 fed by TMA): the
    converged energy must still equal 27 x the primitive cell's to 1e-8 Ha per cell."""
    import dftk_b200 as dftk
    Si = dftk.ElementPsp("Si")
    rep, Ecut, fft, n = 3, 12, 24, 27
    unit = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), symmetries=False)
    bu = dftk.PlaneWaveBasis(unit, Ecut=Ecut, kgrid=(rep, rep, rep), fft_size=(fft, fft, fft))
    ru = dftk.self_consistent_field(bu, tol=1e-9)
    pos = [(np.asarray(p) + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep) for p in POSITIONS]
    sup = dftk.model_DFT(rep * LATTICE, [Si] * (2 * n), pos, functionals=dftk.LDA(), symmetries=False)
    bs = dftk.PlaneWaveBasis(sup, Ecut=Ecut, kgrid=(1, 1, 1), fft_size=(rep * fft,) * 3)
    ctx = bs.architecture.ctx
    ctx.set_option("gemm_backend", 4)
    ctx.set_option("i8_min_rows", 2048)
    try:
        rs = dftk.self_consistent_field(bs, tol=1e-9)
    finally:
        ctx.set_option("gemm_backend", 0)
        ctx.set_option("i8_min_rows", 32768)
    assert rs["converged"] and ru["converged"]
    assert abs(rs["energies"].total - n * ru["energies"].total) < n * 1e-8


def _golden(name):
    import json
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "baseline_configs.json")
    return json.load(open(path))[name]


def _baseline_model(dftk, name):
    if name in ("C1", "C2"):
        return _si_model(dftk, dftk.LDA()), None
    if name == "C4":
        Al = dftk.ElementPsp("Al", functional="pbe")
        pos = [[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]]
        return dftk.model_DFT(7.65339 * np.eye(3), [Al] * 4, pos, functionals=dftk.PBE(), temperature=0.01), dftk.KerkerMixing()
    Fe = dftk.ElementPsp("Fe", functional="pbe")
    lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
    return dftk.model_DFT(lat, [Fe], [[0, 0, 0]], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0]), dftk.KerkerMixing()


@pytest.mark.parametrize("name", ["C1", "C2", "C5", "C4"])
def test_baseline_config_full_size_matches_oracle(name):
    """The BASELINE.json configurations at their STATED sizes (C1: Si2 Ecut 15 k4^3; C2: Si2 Ecut 30 k8^3; C4: Al4 PBE Ecut 40
    k12^3 smearing; C5: Fe bcc PBE collinear Ecut 45 k8^3) against the CPU oracle's converged results of the same
    configuration (tests/golden/baseline_configs.json <- scripts/make_golden_configs.py; the oracle is pinned to the
    reference's golden numbers in tests/test_oracle_golden.py).  BASELINE tolerances: energy 1e-8 Ha/atom, eigenvalues 1e-6 Ha."""
    import dftk_b200 as dftk
    g = _golden(name)
    model, mixing = _baseline_model(dftk, name)
    basis = dftk.PlaneWaveBasis(model, Ecut=g["Ecut"], kgrid=tuple(g["kgrid"]))
    assert list(basis.fft_size) == g["fft_size"] and len(basis.kpoints) == g["n_blocks"]
    res = dftk.self_consistent_field(basis, tol=g["tol"], mixing=mixing)
    assert res["converged"]
    n_at = g["n_atoms"]
    assert abs(res["energies"].total - g["energies"]["total"]) < 1e-8 * n_at
    for term in ("Kinetic", "AtomicLocal", "AtomicNonlocal", "Hartree", "Xc", "Ewald", "PspCorrection"):
        assert abs(res["energies"][term] - g["energies"][term]) < 2e-7 * n_at, term
    if g["temperature"] > 0:
        assert abs(res["eF"] - g["eF"]) < 1e-6
        assert abs(res["energies"]["Entropy"] - g["energies"]["Entropy"]) < 1e-7 * n_at
    nb = g["n_bands_compared"]
    for ik, kpt in enumerate(basis.kpoints):
        jk = [j for j, (kc, sp) in enumerate(zip(g["kcoords"], g["spins"])) if sp == kpt.spin and np.allclose(kc, kpt.coordinate)][0]
        assert abs(basis.kweights[ik] - g["kweights"][jk]) < 1e-13
        np.testing.assert_allclose(res["eigenvalues"][ik][:nb], np.array(g["eigenvalues"][jk][:nb]), atol=1e-6)
    assert abs(float(res["rho"].norm()) * math.sqrt(basis.dvol) - g["rho_l2"]) < 1e-7
    rho_path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "baseline_rho.npz")
    if os.path.exists(rho_path) and name in np.load(rho_path):
        drho = res["rho"].cpu().numpy() - np.load(rho_path)[name]
        assert np.linalg.norm(drho) * math.sqrt(basis.dvol) < 1e-7              # density L2, BASELINE tolerance
    if "magnetisation" in g:
        assert abs(float((res["rho"][0] - res["rho"][1]).sum() * basis.dvol) - g["magnetisation"]) < 1e-5
