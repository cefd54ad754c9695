"""DFT+U on the device: the ortho-atomic orbital table, dftk_b200_orbital_occupation_multi, the Hubbard columns of the
projector products on every H-apply path, the energy/operator consistency and the SCF threading of hubbard_n, against
the NumPy restatement of tests/hubbard_reference.py and the oracle's dense Hamiltonian."""
import numpy as np
import pytest
import torch

import dftk_b200 as dftk
import hubbard_reference as hr
from gpu_common import ctx, device_blocks, silicon_setup, to_dev, rand_psi
from oracle.basis import Element, Model as OModel, PlaneWaveBasis as OBasis
from silicon import LATTICE, POSITIONS
from upf_data import upf_text, product_psp, oracle_psp

pytestmark = pytest.mark.gpu

SI = "Si.pbe-hgh.upf"


def _si_upf():
    return dftk.ElementPsp("Si", product_psp(SI))


def _oracle_orbitals(b):
    return hr.projectors(b, [hr.Orbitals(upf_text(SI), oracle_psp(SI))] * len(b.model.atoms))


def test_orbital_table_matches_oracle():
    kcoords = [[0.0, 0.0, 0.0], [0.1, -0.2, 0.3]]
    model = dftk.model_atomic(LATTICE, [_si_upf()] * 2, POSITIONS, symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=dftk.ExplicitKpoints(kcoords), fft_size=(24, 24, 24))
    projs, labels = dftk.atomic_orbital_projectors(basis)
    om = OModel(LATTICE, [Element("Si", oracle_psp(SI))] * 2, POSITIONS, terms=("Kinetic",), symmetries=False)
    ob = OBasis(om, 10, fft_size=(24, 24, 24), kcoords=kcoords, kweights=[0.5, 0.5])
    oprojs, olabels = _oracle_orbitals(ob)
    assert [(d["iatom"], d["n"], d["l"], d["m"], d["label"]) for d in labels] == olabels
    for P, Q in zip(projs, oprojs):
        P = P.cpu().numpy().T
        assert np.abs(P - Q).max() < 1e-12
        assert np.abs(P.conj().T @ P - np.eye(P.shape[1])).max() < 1e-12


def _blocks_with_orbitals(n_orb, kcoords=((0.1, -0.2, 0.3),), seed=0):
    """Oracle Hamiltonian blocks on the device plus n_orb orthonormal random orbital columns.  At Γ the table is made to
    satisfy Φ(-q) = conj Φ(q) (as the Löwdin orbitals do there), so that the block keeps the folded products."""
    m, b, t, rho, ham = silicon_setup(Ecut=10, fft_size=(24, 24, 24), kcoords=kcoords, kweights=[1.0 / len(kcoords)] * len(kcoords))
    grid, kbs = device_blocks(b, ham)
    rng = np.random.default_rng(seed)
    Phis = []
    for blk, kb in zip(ham, kbs):
        n_G = blk.kpt.n_G
        R = rng.standard_normal((n_G, n_orb)) + 1j * rng.standard_normal((n_G, n_orb))
        if not np.any(blk.kpt.coordinate):
            idx = {tuple(g): i for i, g in enumerate(blk.kpt.G_vectors)}
            R = R + R[[idx[tuple(-g)] for g in blk.kpt.G_vectors]].conj()
        Phi = hr.ortho_lowdin(R)
        Phis.append(Phi)
        kb.set_orbitals(to_dev(Phi.T))
    return b, ham, grid, kbs, Phis


def _herm(n, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))
    return (A + A.conj().T) / 2


def _apply_check(blk, kb, Phi, V, nb=12, tol=1e-12):
    psi = rand_psi(blk.kpt.n_G, nb, seed=3)
    got = kb.apply_h(to_dev(psi)).cpu().numpy().T
    ref = blk.matmul(psi.T) + Phi @ (V @ (Phi.conj().T @ psi.T))
    assert np.abs(got - ref).max() < tol * np.abs(ref).max()


@pytest.mark.parametrize("kcoord,n_orb", [((0.1, -0.2, 0.3), 8), ((0.0, 0.0, 0.0), 8), ((0.0, 0.0, 0.0), 100),
                                          ((0.1, -0.2, 0.3), 100)])
def test_h_apply_complex_and_folded(kcoord, n_orb):
    """Complex products (general k) and the time-reversal fold (Γ); 100 columns pass the batched path's 96 cap."""
    b, ham, grid, kbs, Phis = _blocks_with_orbitals(n_orb, kcoords=(kcoord,))
    blk, kb, Phi = ham[0], kbs[0], Phis[0]
    # Γ keeps the folded products with the orbital columns attached; any other k runs the complex ones
    assert (kb.fold_size() > 0) == (kcoord == (0.0, 0.0, 0.0))
    _apply_check(blk, kb, Phi, np.zeros((n_orb, n_orb)))
    for seed in (1, 2):                       # a second set_orbital_coefficients takes effect
        V = _herm(n_orb, seed)
        kb.set_orbital_coefficients(V)
        _apply_check(blk, kb, Phi, V)


def test_h_apply_folded_gamma_with_ortho_atomic_orbitals():
    """At Γ the Löwdin orbitals keep Φ(-q) = conj Φ(q), so the block stays on the folded products."""
    model = dftk.model_atomic(LATTICE, [_si_upf()] * 2, POSITIONS, symmetries=False,
                              extra_terms=[dftk.Hubbard((dftk.OrbitalManifold("Si", "3P"), 0.1))])
    basis = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=dftk.ExplicitKpoints([[0.0, 0.0, 0.0]]), fft_size=(24, 24, 24))
    term = basis.term("Hubbard")
    assert basis.kblocks[0].n_orb == 6 and basis.kblocks[0].fold_size() > 0
    Phi = term.P_vec[0].cpu().numpy().T
    ip = np.array(basis.kpoints[0].G_vectors.cpu().numpy())
    # Φ(-G) = conj Φ(G)
    idx = {tuple(g): i for i, g in enumerate(ip)}
    mir = np.array([idx[tuple(-g)] for g in ip])
    assert np.abs(Phi[mir] - Phi.conj()).max() < 1e-12 * np.abs(Phi).max()
    rho = dftk.guess_density(basis)
    n0 = [np.zeros((1, 2, 2, 3, 3), dtype=complex)]
    n0[0][0, 0, 0] = n0[0][0, 1, 1] = np.diag([0.3, 0.5, 0.7])
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=rho, hubbard_n=n0)
    _, ham0 = dftk.energy_hamiltonian(basis, None, None, rho=rho)
    psi = to_dev(rand_psi(basis.kpoints[0].n_G, 10, seed=4))
    D = ham[0].hubbard_op.D
    got = (ham[0].mul(psi) - ham0[0].mul(psi)).cpu().numpy().T
    ref = Phi @ (D @ (Phi.conj().T @ psi.cpu().numpy().T))
    assert np.abs(got - ref).max() < 1e-11 * np.abs(ref).max()


@pytest.mark.parametrize("n_orb", [8, 100])
def test_batched_small_solver_sees_the_orbital_term(n_orb):
    """lobpcg_multi on <= 32 bands runs the batched small-matrix path (PD table while n_proj + n_orb <= 96, the
    per-block fallback past it): its eigenvalues are those of the dense H + Φ V Φ', also after a second
    set_orbital_coefficients."""
    kc = ((0.1, -0.2, 0.3), (0.0, 0.0, 0.0))
    b, ham, grid, kbs, Phis = _blocks_with_orbitals(n_orb, kcoords=kc)
    nb = 8
    for round_ in range(2):
        dense = []
        for i, (blk, kb, Phi) in enumerate(zip(ham, kbs, Phis)):
            V = 0.5 * _herm(n_orb, 10 + i + 100 * round_)
            kb.set_orbital_coefficients(V)
            H = blk.matmul(np.eye(blk.kpt.n_G, dtype=complex)) + Phi @ V @ Phi.conj().T
            dense.append(np.linalg.eigvalsh((H + H.conj().T) / 2))
        Xs = [to_dev(rand_psi(blk.kpt.n_G, nb, seed=5 + i)) for i, blk in enumerate(ham)]
        res = dftk.device.lobpcg_multi(kbs, Xs, tol=1e-9, maxiter=300)
        for r, ev in zip(res, dense):
            assert r["converged"]
            assert np.abs(r["λ"] - ev[:nb]).max() < 1e-8


def test_int8_backend_carries_the_orbitals():
    b, ham, grid, kbs, Phis = _blocks_with_orbitals(70)
    blk, kb, Phi = ham[0], kbs[0], Phis[0]
    V = _herm(70, 3)
    c = ctx()
    c.set_option("gemm_backend", 4)
    c.set_option("i8_min_rows", 256)
    try:
        kb.set_orbital_coefficients(V)
        _apply_check(blk, kb, Phi, V, nb=40, tol=1e-12)
        V2 = _herm(70, 4)
        kb.set_orbital_coefficients(V2)
        _apply_check(blk, kb, Phi, V2, nb=40, tol=1e-12)
    finally:
        c.set_option("gemm_backend", 0)
        c.set_option("i8_min_rows", 32768)


@pytest.mark.parametrize("nb", [7, 40])
def test_orbital_occupation_multi(nb):
    """Small (batched projection) and large (per-block GEMM) blocks, both spin channels, against NumPy."""
    kc = ((0.1, -0.2, 0.3), (0.0, 0.0, 0.0), (0.25, 0.0, 0.5))
    b, ham, grid, kbs, Phis = _blocks_with_orbitals(8, kcoords=kc)
    kbs2 = []             # the same blocks (atomic projectors, then the orbital columns), in alternating spin channels
    for i, (blk, kb, Phi) in enumerate(zip(ham, kbs, Phis)):
        P = to_dev(blk.PD[0].T)
        k2 = dftk.KBlock(grid, blk.kpt.mapping, kin=blk.kin, P=P, D=blk.PD[1], spin=i % 2)
        assert k2.n_proj > 0
        k2.set_orbitals(to_dev(Phi.T))
        kbs2.append(k2)
    rng = np.random.default_rng(9)
    psis = [rand_psi(blk.kpt.n_G, nb, seed=20 + i) for i, blk in enumerate(ham)]
    ws = [rng.random(nb) for _ in ham]
    got = dftk.device.orbital_occupation_multi(kbs2, [to_dev(p) for p in psis], ws, 2, 8)
    ref = np.zeros((2, 8, 8), dtype=complex)
    for i, (p, w, Phi) in enumerate(zip(psis, ws, Phis)):
        a = Phi.conj().T @ p.T
        ref[i % 2] += (a * w) @ a.conj().T
    assert np.abs(got - ref).max() < 1e-13 * np.abs(ref).max()


def _hubbard_only_basis(collinear, hub):
    mm = [1.0, 1.0] if collinear else []
    model = dftk.Model(LATTICE, [_si_upf()] * 2, POSITIONS, terms=[hub], magnetic_moments=mm,
                       spin_polarization="collinear" if collinear else "none")
    return dftk.PlaneWaveBasis(model, Ecut=10, kgrid=dftk.MonkhorstPack([1, 2, 3], kshift=[0, 0.5, 0]))


@pytest.mark.parametrize("collinear", [False, True])
@pytest.mark.parametrize("which", ["3P", "3S+3P"])
def test_device_operator_is_the_energy_derivative(which, collinear):
    mans = {"3P": [("3P", 0.01)], "3S+3P": [("3S", 0.01), ("3P", 0.02)]}[which]
    hub = dftk.Hubbard(*[(dftk.OrbitalManifold([0, 1], lab), U) for lab, U in mans])
    basis = _hubbard_only_basis(collinear, hub)
    term = basis.term("Hubbard")
    filled = basis.model.filled_occupation
    rng = np.random.default_rng(0)
    psi, occ = [], []
    for kpt in basis.kpoints:
        q, _ = np.linalg.qr(rng.standard_normal((kpt.n_G, 7)) + 1j * rng.standard_normal((kpt.n_G, 7)))
        psi.append(to_dev(q.T))
        occ.append(filled * np.concatenate([rng.random(4), np.zeros(3)]))
    dpsi = [to_dev(rng.standard_normal(tuple(p.shape)) + 1j * rng.standard_normal(tuple(p.shape))) for p in psi]
    n = dftk.compute_hubbard_n(term, basis, psi, occ)
    E0, ham = dftk.energy_hamiltonian(basis, psi, occ, rho=None, hubbard_n=n)
    assert abs(E0.total - dftk.energy(basis, psi, occ, rho=None, hubbard_n=n).total) < 1e-14

    def E(eps):
        pt = [(p + eps * d).contiguous() for p, d in zip(psi, dpsi)]
        return dftk.energy(basis, pt, occ, rho=None, hubbard_n=dftk.compute_hubbard_n(term, basis, pt, occ)).total

    eps = 1e-6
    diff = (E(eps) - E(-eps)) / (2 * eps)
    pred = 0.0
    for ik in range(len(basis.kpoints)):
        Hp = ham[ik].mul(psi[ik]).cpu().numpy()
        d = dpsi[ik].cpu().numpy()
        pred += 2 * basis.kweights[ik] * np.sum(occ[ik][:4] * np.real(np.sum(d[:4].conj() * Hp[:4], axis=1)))
    assert abs(diff) > 1e-8
    assert abs(diff - pred) < 1e-4 * abs(E0.total) or abs(diff - pred) < 1e-8


def _si_model(hub, **kw):
    extra = [] if hub is None else [hub]
    return dftk.model_DFT(LATTICE, [_si_upf()] * 2, POSITIONS, functionals=dftk.LDA(), extra_terms=extra, **kw)


def test_zero_u_equals_the_model_without_the_term():
    """At one fixed density and orbital set: the same Hψ, energies and eigenpairs with U = 0 as without the term."""
    out = []
    for hub in (None, dftk.Hubbard((dftk.OrbitalManifold("Si", "3P"), 0.0))):
        basis = dftk.PlaneWaveBasis(_si_model(hub), Ecut=12, kgrid=(2, 2, 2))
        rho = dftk.guess_density(basis)
        psi = [to_dev(rand_psi(k.n_G, 8, seed=30 + ik)) for ik, k in enumerate(basis.kpoints)]
        psi = [torch.linalg.qr(p.T)[0].T.contiguous() for p in psi]
        occ = [np.array([2.0] * 4 + [0.0] * 4) for _ in basis.kpoints]
        n = None if hub is None else dftk.compute_hubbard_n(basis.term("Hubbard"), basis, psi, occ)
        E, ham = dftk.energy_hamiltonian(basis, psi, occ, rho=rho, hubbard_n=n)
        Hpsi = [ham[ik].mul(p).cpu().numpy() for ik, p in enumerate(psi)]
        eig = [ham[ik].bind().lobpcg(p.clone(), tol=1e-10, maxiter=300)["λ"] for ik, p in enumerate(psi)]
        out.append((E, Hpsi, eig))
    (E0, H0, l0), (E1, H1, l1) = out
    assert E1["Hubbard"] == 0.0
    assert abs(E1.total - E0.total) < 1e-12
    for a, b in zip(H1, H0):
        assert np.abs(a - b).max() < 1e-12 * np.abs(b).max()
    for a, b in zip(l1, l0):
        assert np.abs(a - b).max() < 1e-12


def _oracle_scf_pair(U, tol, **kw):
    """Package SCF and the NumPy restatement's SCF (oracle Hamiltonian + Hubbard operator) of Si2, U on 3P."""
    hub = dftk.Hubbard((dftk.OrbitalManifold("Si", "3P"), U))
    basis = dftk.PlaneWaveBasis(_si_model(hub, **kw), Ecut=10, kgrid=(2, 2, 2))
    res = dftk.self_consistent_field(basis, tol=tol, seed=1, maxiter=100)
    assert res["converged"]
    okw = dict(temperature=kw.get("temperature", 0.0), smearing=kw.get("smearing"),
               magnetic_moments=kw.get("magnetic_moments", ()))
    om = OModel(LATTICE, [Element("Si", oracle_psp(SI))] * 2, POSITIONS, **okw)
    ob = OBasis(om, 10, kgrid=(2, 2, 2))
    assert ob.fft_size == basis.fft_size and len(ob.kpoints) == len(basis.kpoints)
    ores = hr.scf(ob, [hr.Orbitals(upf_text(SI), oracle_psp(SI))] * 2, [hr.Manifold([0, 1], 1, 1, U)], tol=tol)
    assert ores["converged"]
    return basis, res, ob, ores


def _compare_with_oracle(basis, res, ob, ores):
    """BASELINE tolerances: energy 1e-8 Ha/atom, eigenvalues 1e-6 Ha, density L2 1e-7; n 1e-7 and the Hubbard energy."""
    n_atoms = 2
    assert abs(res["energies"].total - ores["energies"]["total"]) < 1e-8 * n_atoms
    assert abs(res["energies"]["Hubbard"] - ores["energies"]["Hubbard"]) < 1e-8 * n_atoms
    assert res["energies"]["Hubbard"] > 1e-3
    for ik, kpt in enumerate(basis.kpoints):
        jk = [j for j, ok in enumerate(ob.kpoints) if np.allclose(ok.coordinate, kpt.coordinate) and ok.spin == kpt.spin][0]
        np.testing.assert_allclose(res["eigenvalues"][ik][:4], ores["eigenvalues"][jk][:4], atol=1e-6)
    drho = res["rho"].cpu().numpy() - ores["rho"]
    assert np.linalg.norm(drho) * np.sqrt(basis.dvol) < 1e-7
    assert np.abs(res["hubbard_n"][0] - ores["hubbard_n"][0]).max() < 1e-7


def test_scf_with_hubbard_matches_oracle():
    """Case (a): Si2 with Si.pbe-hgh.upf, U on 3P, against the restatement's SCF built on the oracle."""
    basis, res, ob, ores = _oracle_scf_pair(0.2, 1e-10)
    _compare_with_oracle(basis, res, ob, ores)
    term = basis.term("Hubbard")
    n = res["hubbard_n"]
    # the occupation of the final orbitals, recomputed (copies: no cached sum), is the returned one: it is never mixed
    again = dftk.compute_hubbard_n(term, basis, [p.clone() for p in res["psi"]], [np.array(o) for o in res["occupation"]])
    assert np.abs(again[0] - n[0]).max() < 1e-12
    # the energy and the operator coefficients against the restatement at the same n
    D, E = term.coefficients(basis, n)
    Eo, Do = hr.energy_and_coefficients(ob, [hr.Manifold([0, 1], 1, 1, 0.2)], n)
    assert abs(E - Eo) < 1e-14 and np.abs(D - Do).max() < 1e-14
    assert abs(E - res["energies"]["Hubbard"]) < 1e-14
    with pytest.raises(NotImplementedError, match="Hubbard"):
        dftk.compute_forces(res)


def test_atomic_orbital_projections():
    basis = dftk.PlaneWaveBasis(_si_model(None), Ecut=10, kgrid=(2, 2, 2))
    psi = [to_dev(rand_psi(k.n_G, 5, seed=40 + ik)) for ik, k in enumerate(basis.kpoints)]
    proj, labels = dftk.atomic_orbital_projections(basis, psi)
    tables, labels2 = dftk.atomic_orbital_projectors(basis)
    assert labels == labels2 and len(labels) == 8
    for P, Phi, p in zip(proj, tables, psi):
        ref = np.abs(p.cpu().numpy().conj() @ Phi.cpu().numpy().T) ** 2
        assert P.shape == (5, 8) and np.abs(P - ref).max() < 1e-12 * ref.max()


def test_two_rank_sharded_hubbard_scf_matches_single_gpu():
    """World size 2: the k-sharded SCF (the occupation partials travel in the density allreduce) equals one GPU."""
    import json, os, subprocess, sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29537",
                        os.path.join(root, "scripts", "hubbard_multi_gpu_check.py")], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("MULTIGPU_RESULT ")][-1][len("MULTIGPU_RESULT "):])
    assert out["nk_local"] < out["nk_total"]
    assert out["dE"] < 1e-10 and out["dn"] < 1e-10, out


def test_spin_polarised_scf_maps_atoms_onto_each_other():
    """Case (b): collinear Si2 with Gaussian smearing and U on 3P against the restatement's SCF; the inversion of the
    diamond structure exchanges the two atoms, so the symmetrisation permutes the atom blocks while it rotates them.
    (The vendored Tl.pbe-d-hgh.upf carries all-zero PP_CHI tables, which the Löwdin step rejects as linearly dependent,
    so no d manifold is run here; the l = 2 Wigner matrices are pinned on the host.)"""
    kw = dict(temperature=0.01, smearing="Gaussian", magnetic_moments=[1.0, 1.0])
    model = _si_model(None, **kw)
    moved = [s.W @ POSITIONS[0] + s.w - POSITIONS[1] for s in model.symmetries]
    assert any(np.allclose(d, np.round(d), atol=1e-8) for d in moved)       # a symmetry maps atom 0 onto atom 1
    basis, res, ob, ores = _oracle_scf_pair(0.3, 1e-10, **kw)
    n = res["hubbard_n"][0]
    assert n.shape == (2, 2, 2, 3, 3)
    assert np.abs(n - n.conj().transpose(0, 1, 2, 4, 3)).max() < 1e-12
    assert np.abs(n[:, 0, 1]).max() == 0.0
    _compare_with_oracle(basis, res, ob, ores)
