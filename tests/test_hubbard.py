"""DFT+U on the host: PP_PSWFC parsing, Wigner matrices, manifold resolution, and the NumPy restatement of the Hubbard
term (tests/hubbard_reference.py) against the reference's identities (test/hubbard.jl, test/hamiltonian_consistency.jl)."""
import numpy as np
import pytest

import dftk_b200 as dftk
from dftk_b200.pseudo import PspHgh
import hubbard_reference as hr
from oracle.basis import Element, Model as OModel, PlaneWaveBasis as OBasis, SymOp
from silicon import LATTICE, POSITIONS
from upf_data import upf_text, product_psp, oracle_psp

CHI = {"Si.pbe-hgh.upf": [("3S", 0), ("3P", 1)], "Tl.pbe-d-hgh.upf": [("6S", 0), ("6P", 1), ("5D", 2)],
       "C_m.upf": [("2S", 0), ("2P", 1)], "Al_m.upf": [("3S", 0), ("3P", 1)]}


@pytest.mark.parametrize("name", sorted(CHI))
def test_pswfc_parsing_matches_the_file(name):
    psp = product_psp(name)
    got = [(psp.pswfc_label(i, l), l) for l in range(psp.lmax + 1) for i in range(1, psp.count_n_pswfc_radial(l) + 1)]
    assert got == CHI[name]
    in_file = [(lab, l) for lab, l, _, _ in hr.parse_pswfc(upf_text(name)) if l <= psp.lmax]
    assert sorted(got) == sorted(in_file)
    assert psp.count_n_pswfc() == sum(2 * l + 1 for _, l in CHI[name])
    assert psp.count_n_pswfc_radial() == len(CHI[name])
    for lab, l in CHI[name]:
        assert psp.find_pswfc(lab)[0] == l
    with pytest.raises(ValueError, match="Could not find"):
        psp.find_pswfc("9G")
    r = psp.rgrid
    rchi = {lab: f for lab, _, _, f in hr.parse_pswfc(upf_text(name))}
    for lab, l in CHI[name]:
        i = psp.find_pswfc(lab)[1]
        np.testing.assert_array_equal(psp.r2_pswfcs[l][i - 1], r * rchi[lab][:len(r)])


def test_hgh_has_no_atomic_wavefunctions():
    psp = dftk.load_psp("Si", "lda")
    assert isinstance(psp, PspHgh)
    with pytest.raises(ValueError, match="does not implement atomic wavefunctions"):
        psp.count_n_pswfc()


WIGNER = [
    (np.eye(3), np.eye(3), np.eye(5)),
    (-np.eye(3), -np.eye(3), np.eye(5)),
    (np.diag([1.0, -1, -1]), np.diag([-1.0, -1, 1]), np.diag([-1.0, 1, 1, -1, 1])),
    (np.array([[0.0, 1, 0], [1, 0, 0], [0, 0, 1]]), np.array([[0.0, 0, 1], [0, 1, 0], [1, 0, 0]]),
     np.array([[1.0, 0, 0, 0, 0], [0, 0, 0, 1, 0], [0, 0, 1, 0, 0], [0, 1, 0, 0, 0], [0, 0, 0, 0, -1]])),
]


@pytest.mark.parametrize("W,Dp,Dd", WIGNER)
def test_wigner_d_matrix_known_cases(W, Dp, Dd):
    np.testing.assert_allclose(dftk.wigner_d_matrix(1, W), Dp, atol=1e-12)
    np.testing.assert_allclose(dftk.wigner_d_matrix(2, W), Dd, atol=1e-12)


def test_wigner_d_matrix_is_a_representation():
    rng = np.random.default_rng(3)
    Q1, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    Q2, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    for l in (1, 2, 3):
        D12 = dftk.wigner_d_matrix(l, Q1 @ Q2)
        np.testing.assert_allclose(D12, dftk.wigner_d_matrix(l, Q1) @ dftk.wigner_d_matrix(l, Q2), atol=1e-11)
        np.testing.assert_allclose(dftk.wigner_d_matrix(l, Q1), hr.wigner_d_matrix(l, Q1), atol=1e-11)


def _nio_like():
    """Two Tl and two Si on the NiO rocksalt positions (test/hubbard.jl:44-77 with vendored pseudopotentials)."""
    a = 7.9
    lat = a * np.array([[1.0, 0.5, 0.5], [0.5, 1.0, 0.5], [0.5, 0.5, 1.0]])
    Tl = dftk.ElementPsp("Tl", product_psp("Tl.pbe-d-hgh.upf"))
    Si = dftk.ElementPsp("Si", product_psp("Si.pbe-hgh.upf"))
    pos = [[0.0, 0, 0], [0.25, 0.25, 0.25], [0.5, 0.5, 0.5], [0.75, 0.75, 0.75]]
    return dftk.model_DFT(lat, [Tl, Si, Tl, Si], pos, functionals=dftk.PBE()), Tl, Si


def test_manifold_resolution_forms():
    model, Tl, _ = _nio_like()
    for man in [dftk.OrbitalManifold(Tl, "5D"), dftk.OrbitalManifold("Tl", "5D"), dftk.OrbitalManifold(Tl, (2, 1)),
                dftk.OrbitalManifold("Tl", (2, 1)), dftk.OrbitalManifold([0, 2], "5D")]:
        r = dftk.resolve_hubbard_manifold(man, model)
        assert r.psp is Tl.psp and r.iatoms == [0, 2] and (r.l, r.i) == (2, 1)


def test_manifold_resolution_errors():
    model, Tl, Si = _nio_like()
    with pytest.raises(ValueError, match="no atoms"):
        dftk.resolve_hubbard_manifold(dftk.OrbitalManifold("Fe", "3D"), model)
    with pytest.raises(ValueError, match="multiple psps"):
        dftk.resolve_hubbard_manifold(dftk.OrbitalManifold([0, 1], "5D"), model)
    with pytest.raises(ValueError, match="symmetries"):
        dftk.resolve_hubbard_manifold(dftk.OrbitalManifold([0], "5D"), model)
    with pytest.raises(ValueError, match="Could not find"):
        dftk.resolve_hubbard_manifold(dftk.OrbitalManifold("Tl", "3D"), model)

    class NoPsp:
        symbol = "X"
        psp = None
    m2, _, _ = _nio_like()
    m2.atoms = [NoPsp()] + m2.atoms[1:]
    with pytest.raises(ValueError, match="must have a psp"):
        dftk.resolve_hubbard_manifold(dftk.OrbitalManifold([0], (0, 1)), m2)
    # a manifold that is not closed under the symmetries is fine once the model has none
    m3 = dftk.model_DFT(model.lattice, model.atoms, model.positions, functionals=dftk.PBE(), symmetries=False)
    assert dftk.resolve_hubbard_manifold(dftk.OrbitalManifold([0], "5D"), m3).iatoms == [0]


def test_hubbard_constructors():
    m1, m2 = dftk.OrbitalManifold("Si", "3S"), dftk.OrbitalManifold("Si", "3P")
    a = dftk.Hubbard([m1, m2], [0.01, 0.02])
    b = dftk.Hubbard((m1, 0.01), (m2, 0.02))
    assert a.U == b.U == [0.01, 0.02] and a.manifolds == b.manifolds
    with pytest.raises(ValueError, match="must match"):
        dftk.Hubbard([m1, m2], [0.01])
    Si = dftk.ElementPsp("Si", product_psp("Si.pbe-hgh.upf"))
    model = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), extra_terms=[a])
    assert model.term_names[-1] == "Hubbard" and model.term_types[-1] is a


# ------------------------------------------------------------------ the NumPy restatement
def _oracle_silicon(collinear, symmetries=True, kgrid=(1, 2, 3), kshift=(0, 0.5, 0), Ecut=10):
    text = upf_text("Si.pbe-hgh.upf")
    psp = oracle_psp("Si.pbe-hgh.upf")
    Si = Element("Si", psp)
    mm = [1.0, 1.0] if collinear else ()
    m = OModel(LATTICE, [Si, Si], POSITIONS, terms=("Kinetic",), magnetic_moments=mm, symmetries=symmetries)
    b = OBasis(m, Ecut, kgrid=kgrid, kshift=kshift)
    orbs = [hr.Orbitals(text, psp)] * 2
    return m, b, orbs


def _random_state(b, n_bands=4, n_empty=3, seed=0):
    rng = np.random.default_rng(seed)
    psi, occ = [], []
    filled = b.model.filled_occupation
    for kpt in b.kpoints:
        q, _ = np.linalg.qr(rng.standard_normal((kpt.n_G, n_bands + n_empty)) + 1j * rng.standard_normal((kpt.n_G, n_bands + n_empty)))
        psi.append(q)
        occ.append(filled * np.concatenate([rng.random(n_bands), np.zeros(n_empty)]))
    return psi, occ


def test_oracle_orbitals_are_orthonormal():
    _, b, orbs = _oracle_silicon(False)
    projs, labels = hr.projectors(b, orbs)
    assert len(labels) == 2 * 4
    for P in projs:
        assert np.abs(P.conj().T @ P - np.eye(P.shape[1])).max() < 1e-12


MANIFOLDS = {"3P": [((1, 1), 0.01)], "3S+3P": [((0, 1), 0.01), ((1, 1), 0.02)]}


@pytest.mark.parametrize("collinear", [False, True])
@pytest.mark.parametrize("which", sorted(MANIFOLDS))
def test_oracle_operator_is_the_energy_derivative(which, collinear):
    """hamiltonian_consistency.jl: 2 Σ_k w_k Σ_n f_n Re<δψ_n|H_U ψ_n> equals the central difference of E_U."""
    _, b, orbs = _oracle_silicon(collinear)
    mans = [hr.Manifold([0, 1], l, i, U) for (l, i), U in MANIFOLDS[which]]
    projs, labels = hr.projectors(b, orbs)
    Phi = hr.manifold_table(projs, labels, mans)
    psi, occ = _random_state(b)
    rng = np.random.default_rng(1)
    dpsi = [rng.standard_normal(p.shape) + 1j * rng.standard_normal(p.shape) for p in psi]

    def E(eps):
        pt = [p + eps * d for p, d in zip(psi, dpsi)]
        return hr.energy_and_coefficients(b, mans, [hr.hubbard_n(b, projs, labels, m, pt, occ) for m in mans])[0]

    E0, D = hr.energy_and_coefficients(b, mans, [hr.hubbard_n(b, projs, labels, m, psi, occ) for m in mans])
    eps = 1e-6
    diff = (E(eps) - E(-eps)) / (2 * eps)
    pred = 0.0
    for ik, kpt in enumerate(b.kpoints):
        Hpsi = Phi[ik] @ (D[kpt.spin] @ (Phi[ik].conj().T @ psi[ik]))
        pred += 2 * b.kweights[ik] * np.sum(occ[ik][:4] * np.real(np.sum(dpsi[ik][:, :4].conj() * Hpsi[:, :4], axis=0)))
    assert abs(diff) > 1e-8
    assert abs(diff - pred) < 1e-4 * abs(E0) or abs(diff - pred) < 1e-8


def _ground_state_occupations(b):
    """Orbitals of the oracle's atomic Hamiltonian (dense diagonalisation, four filled bands per k)."""
    from oracle.terms import Terms, energy_hamiltonian, guess_density
    _, ham = energy_hamiltonian(b, Terms(b), None, None, guess_density(b))
    psi, occ = [], []
    for blk in ham:
        H = blk.matmul(np.eye(blk.kpt.n_G, dtype=complex))
        _, V = np.linalg.eigh((H + H.conj().T) / 2)
        psi.append(V[:, :4])
        occ.append(np.full(4, 2.0))
    return psi, occ


def test_oracle_symmetrised_ibz_equals_full_bz():
    """test/hubbard.jl:121-131: n from the irreducible wedge, symmetrised, equals n from the whole zone."""
    psp = oracle_psp("Si.pbe-hgh.upf")
    text = upf_text("Si.pbe-hgh.upf")
    Si = Element("Si", psp)
    out = []
    for reduce in (True, False):
        m = OModel(LATTICE, [Si, Si], POSITIONS, terms=("Kinetic", "AtomicLocal", "AtomicNonlocal"), symmetries=True)
        b = OBasis(m, 6, kgrid=(2, 2, 2), use_symmetries_for_kpoint_reduction=reduce)
        projs, labels = hr.projectors(b, [hr.Orbitals(text, psp)] * 2)
        psi, occ = _ground_state_occupations(b)
        man = hr.Manifold([0, 1], 1, 1, 0.1)
        syms = None if reduce else [SymOp(np.eye(3), np.zeros(3))]      # the whole zone needs no symmetrisation
        out.append((len(b.kpoints), hr.hubbard_n(b, projs, labels, man, psi, occ, symmetries=syms)))
    assert out[0][0] < out[1][0]
    np.testing.assert_allclose(out[0][1], out[1][1], atol=1e-10)
