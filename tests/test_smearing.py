"""Marzari-Vanderbilt and Methfessel-Paxton smearing, the two-stage Fermi-level search and the kinetic blow-ups of
energy-cutoff smearing (CPU): the reference's smearing identities and pinned Fermi levels (test/occupation.jl), the
blow-up's regularity, the model's argument checks, and oracle forces at cold smearing against the free energy."""
import json
import math
import os
import warnings
from types import SimpleNamespace

import numpy as np
import pytest

import smearing_oracle as so
from silicon import LATTICE

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "smearing", "fermi_levels.json")
KINDS = ["None", "FermiDirac", "Gaussian", "MarzariVanderbilt"] + [("MethfesselPaxton", n) for n in range(1, 5)]


def _product():
    from dftk_b200 import terms
    return SimpleNamespace(occupation=terms.smearing_occupation, entropy=terms.smearing_entropy,
                           occupation_derivative=terms.occupation_derivative)


@pytest.mark.parametrize("impl", ["product", "oracle"])
@pytest.mark.parametrize("kind", KINDS, ids=str)
def test_smearing_identities(kind, impl):
    """test/occupation.jl:17-33: the limits at ±∞, f' against a finite difference and s'(x) = x f'(x)."""
    S = _product() if impl == "product" else so
    assert S.occupation(kind, -np.inf) == 1 and S.occupation(kind, np.inf) == 0
    x, h = 0.04, 1e-8
    fprime = (S.occupation(kind, x + h) - S.occupation(kind, x)) / h
    assert abs(fprime - S.occupation_derivative(kind, x)) < 1e-4
    sprime = (S.entropy(kind, x + h) - S.entropy(kind, x)) / h
    assert abs(sprime - x * fprime) < 1e-4
    # the closed-form derivative over a range of x, against a central difference
    xs = np.linspace(-4, 4, 81)
    cd = (S.occupation(kind, xs + 1e-6) - S.occupation(kind, xs - 1e-6)) / 2e-6
    np.testing.assert_allclose(S.occupation_derivative(kind, xs), cd if kind != "None" else 0 * xs, atol=1e-8)


@pytest.mark.parametrize("kind", KINDS + [("MethfesselPaxton", 0), ("MethfesselPaxton", 7)], ids=str)
def test_product_smearing_matches_oracle(kind):
    S = _product()
    x = np.linspace(-7, 7, 141)
    for a, b in [(S.occupation, so.occupation), (S.entropy, so.entropy),
                 (S.occupation_derivative, so.occupation_derivative)]:
        np.testing.assert_allclose(a(kind, x), b(kind, x), rtol=1e-12, atol=1e-14)
    # order 0 is Gaussian smearing
    np.testing.assert_allclose(S.occupation(("MethfesselPaxton", 0), x), S.occupation("Gaussian", x), atol=1e-16)


def _fermi_cases():
    d = json.load(open(GOLDEN))
    out = []
    for name, case in d.items():
        for kind, T, ref in case["cases"]:
            for alg in case["fermialgs"]:
                out.append(pytest.param(name, tuple(kind) if isinstance(kind, list) else kind, T, ref, alg,
                                        id=f"{name}-{kind}-{T}-{alg}"))
    return out


def _setups():
    """The two bases of test/occupation.jl: Mg atoms in the silicon lattice on a shifted 2x3x4 grid, and spin-polarised
    bcc iron on 4x4x4.  Returns model, irreducible k-points and weights of the port, and the symmetries used."""
    import dftk_b200 as dftk
    from dftk_b200.basis import irreducible_kcoords, compute_fft_size, _kkey
    from dftk_b200.model import SYMMETRY_TOLERANCE
    fe_psp = dftk.load_psp(os.path.join(os.path.dirname(__file__), "golden", "iron_lda", "Fe-q8.hgh"))
    si_psp = dftk.load_psp("Si")
    out = {}
    for name in ("simple_metal", "multiple_fermi_levels"):
        s = json.load(open(GOLDEN))[name]["setup"]
        if name == "simple_metal":
            Mg = dftk.ElementPsp("Mg", psp=si_psp)        # only the species label enters the symmetry search
            model = dftk.Model(LATTICE, [Mg, Mg], s["positions"], n_electrons=4, temperature=1e-2)
        else:
            lat = s["lattice_bcc_a"] * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]])
            model = dftk.Model(lat, [dftk.ElementPsp("Fe", psp=fe_psp)], s["positions"], n_electrons=8,
                               temperature=1e-2, magnetic_moments=s["magnetic_moments"])
        kgrid = dftk.MonkhorstPack(s["kgrid"], kshift=s["kshift"])
        # the symmetries PlaneWaveBasis keeps: compatible with the real-space grid and with the k-grid
        from fractions import Fraction
        dens = {Fraction(float(wi)).limit_denominator(12).denominator for sy in model.symmetries for wi in sy.w}
        n = np.array(compute_fft_size(model, s["Ecut"], 2.0, tuple(sorted({2, 3, 4, 6} & dens)) or (1,)))
        syms = [sy for sy in model.symmetries if np.all(np.abs(sy.w * n - np.round(sy.w * n)) / n <= SYMMETRY_TOLERANCE)]
        keys = {_kkey(k) for k in kgrid.reducible_kcoords()}
        syms = [sy for sy in syms if all(_kkey(sy.S @ k) in keys for k in kgrid.reducible_kcoords())]
        k, w = irreducible_kcoords(kgrid, syms)
        out[name] = (model, k, w, syms)
    return out


@pytest.fixture(scope="module")
def setups():
    return _setups()


def _paired_weights(setup, case):
    """Weights of the fixture's eigenvalue rows.  The rows follow the reference's k-point order (spglib's irreducible
    mesh: representatives by ascending grid index, spin-major); each fixture k-point is matched to the port's
    symmetry-equivalent irreducible point, and its degeneracy pattern is checked against that point's site symmetry."""
    from dftk_b200.basis import _kkey
    model, kirr, wirr, syms = setup
    weights = []
    for k in case["kcoords"]:
        hits = [w for kp, w in zip(kirr, wirr) if any(_kkey(s.S @ kp) == _kkey(k) for s in syms)]
        assert len(hits) == 1, k
        weights.append(hits[0])
    n_spin = model.n_spin_components
    assert len(case["eigenvalues"]) == n_spin * len(weights)
    for row, e in enumerate(case["eigenvalues"]):
        k = np.array(case["kcoords"][row % len(weights)])
        little = [s for s in syms if _kkey(s.S @ k) == _kkey(k)]
        abelian = all(np.array_equal(a.S @ b.S, b.S @ a.S) for a in little for b in little)
        e = np.asarray(e)
        groups = np.split(e, np.nonzero(np.diff(e) > 1e-6)[0] + 1)
        deg = max(len(g) for g in groups)
        if deg >= 3:
            assert len(little) >= 24, (row, k)       # a 3-dimensional irrep needs a cubic site group
        if deg == 2 and n_spin == 2:
            assert not abelian, (row, k)
        if len(little) >= 24:
            assert deg >= 3, (row, k)
        if abelian and n_spin == 2:
            assert deg == 1, (row, k)
    return weights * n_spin


@pytest.mark.parametrize("name,kind,T,ref,alg", _fermi_cases())
def test_pinned_fermi_levels(setups, name, kind, T, ref, alg):
    """test/occupation.jl:110-149 ("Smearing for a simple metal", both algorithms) and :151-207 ("Fermi level finding
    for smearing multiple εF", the default algorithm): the electron count and εF ≈ the reference's (rtol 1.5e-8, Julia's
    ≈).  MP(2) and MP(5) at T = 1e-2 have a second root with positive DOS; the pinned one must be found."""
    import dftk_b200 as dftk
    from dftk_b200.occupation import compute_occupation
    case = json.load(open(GOLDEN))[name]
    setup = setups[name]
    model0, kirr, wirr, _ = setup
    assert len(kirr) == {"simple_metal": 12, "multiple_fermi_levels": 8}[name]
    assert abs(sum(wirr) - 1) < 1e-14
    w = _paired_weights(setup, case)
    model = dftk.Model(model0.lattice, model0.atoms, model0.positions, n_electrons=model0.n_electrons, temperature=T,
                       smearing=kind, magnetic_moments=model0.magnetic_moments)
    basis = SimpleNamespace(model=model, kweights=w, comm_kpts=dftk.KpointComm())
    fermialg = {"FermiBisection": dftk.FermiBisection(), "FermiTwoStage": dftk.FermiTwoStage(), "default": None}[alg]
    eig = [np.array(e) for e in case["eigenvalues"]]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        occ, eF = compute_occupation(basis, eig, fermialg=fermialg, tol_n_elec=case["tol_n_elec"])
    assert abs(sum(wk * o.sum() for wk, o in zip(w, occ)) - model.n_electrons) <= 1.5e-8 * model.n_electrons
    assert eF == pytest.approx(ref, rel=1.5e-8)
    # the oracle finds the same Fermi level
    eF_o = so.fermi_level(model, w, eig, {"FermiBisection": "bisection", "FermiTwoStage": "two-stage",
                                          "default": None}[alg], tol_n_elec=case["tol_n_elec"])
    assert eF_o == pytest.approx(ref, rel=1.5e-8)


def test_negative_dos_warning_at_the_pinned_root(setups):
    """MP(2) at T = 1e-2 lands on the root with negative DOS: compute_occupation says so (occupation.jl:87-99)."""
    import dftk_b200 as dftk
    from dftk_b200.occupation import compute_occupation
    case = json.load(open(GOLDEN))["multiple_fermi_levels"]
    m0 = setups["multiple_fermi_levels"][0]
    w = _paired_weights(setups["multiple_fermi_levels"], case)
    eig = [np.array(e) for e in case["eigenvalues"]]
    for kind, expect in [(("MethfesselPaxton", 2), True), ("MarzariVanderbilt", False)]:
        model = dftk.Model(m0.lattice, m0.atoms, m0.positions, n_electrons=8, temperature=1e-2, smearing=kind,
                           magnetic_moments=[4])
        with warnings.catch_warnings(record=True) as got:
            warnings.simplefilter("always")
            compute_occupation(SimpleNamespace(model=model, kweights=w, comm_kpts=dftk.KpointComm()), eig)
        assert any("Negative density of states" in str(g.message) for g in got) == expect


def test_default_fermialg_keeps_bisection_for_monotone_smearing():
    import dftk_b200 as dftk
    from dftk_b200.occupation import compute_occupation
    assert isinstance(dftk.default_fermialg("FermiDirac"), dftk.FermiBisection)
    assert isinstance(dftk.default_fermialg("Gaussian"), dftk.FermiBisection)
    assert isinstance(dftk.default_fermialg("MarzariVanderbilt"), dftk.FermiTwoStage)
    assert isinstance(dftk.default_fermialg(("MethfesselPaxton", 1)), dftk.FermiTwoStage)
    Si = dftk.ElementPsp("Si")
    rng = np.random.default_rng(1)
    eig = [np.sort(rng.normal(0.2, 0.3, 9)) for _ in range(20)]
    w = list(rng.random(20))
    w = [x / sum(w) for x in w]
    for kind in ("FermiDirac", "Gaussian"):
        m = dftk.model_DFT(LATTICE, [Si, Si], [np.ones(3) / 8, -np.ones(3) / 8], functionals=dftk.LDA(),
                           temperature=0.01, smearing=kind)
        b = SimpleNamespace(model=m, kweights=w, comm_kpts=dftk.KpointComm())
        occ0, eF0 = compute_occupation(b, eig)
        occ1, eF1 = compute_occupation(b, eig, fermialg=dftk.FermiBisection())
        assert eF0 == eF1 and all(np.array_equal(a, c) for a, c in zip(occ0, occ1))


def test_blowup_regularity():
    """kinetic.jl:63-110: the factor is 1 below x = 0.85 (CHV) and below |p| = sqrt(2 (Ecut - Ecutsm)) (Abinit),
    Ekin · factor is C² across CHV's interpolation window and continuous at Abinit's; product and oracle agree."""
    import dftk_b200 as dftk
    import torch
    Ecut = 5.0
    pmax = math.sqrt(2 * Ecut)
    chv, ab = dftk.BlowupCHV(), dftk.BlowupAbinit()
    p = np.linspace(0, 0.8499 * pmax, 200)
    assert np.all(chv(p, Ecut) == 1)
    p = np.linspace(0, math.sqrt(2 * (Ecut - 0.5 * Ecut)), 200)
    assert np.all(ab(p, Ecut) == 1)
    def derivatives(blow, p, h=1e-5):
        E = lambda q: q ** 2 / 2 * blow(q, Ecut)
        return E(p), (E(p + h) - E(p - h)) / (2 * h), (E(p + h) - 2 * E(p) + E(p - h)) / h ** 2

    # CHV: Ekin · factor and its first two derivatives are continuous across [0.85, 0.90] sqrt(2 Ecut)
    p = np.linspace(0.83 * pmax, 0.92 * pmax, 2001)
    dp = p[1] - p[0]
    E, d1, d2 = derivatives(chv, p)
    assert np.max(np.abs(np.diff(E))) < 1.01 * dp * np.max(np.abs(d1))
    assert np.max(np.abs(np.diff(d1))) < 1.01 * dp * np.max(np.abs(d2))
    assert np.max(np.abs(np.diff(d2))) < 0.05 * np.max(np.abs(d2))
    # Abinit: continuous at the window's lower edge.  The reference's polynomial x²(3 + x - 6x² + 3x²) has slope -3 at
    # x = 1, so the first derivative of Ekin · factor jumps there; it is restated as written.
    p0 = math.sqrt(2 * (Ecut - 0.5 * Ecut))
    E, d1, _ = derivatives(ab, np.array([p0 - 1e-3, p0 + 1e-3]))
    assert abs(E[1] - E[0]) < 1e-2
    assert d1[0] == pytest.approx(p0 - 1e-3, rel=1e-6) and d1[1] < 0
    for blow in (chv, ab):       # the torch path (used for the device table) gives the same factor
        p = np.linspace(0, 0.99 * pmax, 301)
        np.testing.assert_allclose(blow(torch.tensor(p), Ecut).numpy(), blow(p, Ecut), rtol=1e-15)
    p = np.linspace(0, 0.999 * pmax, 5001)
    np.testing.assert_allclose(chv(p, Ecut), so.blowup_chv(p, Ecut), rtol=1e-13)
    np.testing.assert_allclose(ab(p, Ecut), so.blowup_abinit(p, Ecut), rtol=1e-13)
    np.testing.assert_allclose(dftk.BlowupAbinit(0.3)(p, Ecut), so.blowup_abinit(p, Ecut, 0.3), rtol=1e-13)
    with pytest.raises(AssertionError):
        dftk.BlowupAbinit(1.0)(p, Ecut)
    with pytest.raises(AssertionError):
        so.blowup_abinit(p, Ecut, 1.0)


def test_model_arguments():
    import dftk_b200 as dftk
    Si = dftk.ElementPsp("Si")
    pos = [np.ones(3) / 8, -np.ones(3) / 8]
    for kind in ("None", "FermiDirac", "Gaussian", "MarzariVanderbilt"):
        assert dftk.Model(LATTICE, [Si, Si], pos, temperature=0.01, smearing=kind).smearing == kind
    assert dftk.Model(LATTICE, [Si, Si], pos, temperature=0.01).smearing == "FermiDirac"
    assert dftk.Model(LATTICE, [Si, Si], pos).smearing == "None"
    assert dftk.Model(LATTICE, temperature=0.01, smearing=("MethfesselPaxton", 2)).smearing == ("MethfesselPaxton", 2)
    assert dftk.Model(LATTICE, temperature=0.01, smearing=["MethfesselPaxton", np.int64(0)]).smearing == ("MethfesselPaxton", 0)
    for bad in (("MethfesselPaxton", -1), ("MethfesselPaxton", 1.5), ("MethfesselPaxton", True), ("MethfesselPaxton", "1")):
        with pytest.raises(ValueError):
            dftk.Model(LATTICE, temperature=0.01, smearing=bad)
    for bad in ("Cold", "MethfesselPaxton", ("MarzariVanderbilt", 1), ("MethfesselPaxton",)):
        with pytest.raises(NotImplementedError):
            dftk.Model(LATTICE, temperature=0.01, smearing=bad)
    m = dftk.model_DFT(LATTICE, [Si, Si], pos, functionals=dftk.LDA(), kinetic_blowup=dftk.BlowupCHV())
    assert m.term_names[0] == "Kinetic" and isinstance(m.term_types[0], dftk.Kinetic)
    assert isinstance(m.term_types[0].blowup, dftk.BlowupCHV) and m.term_types[0].scaling_factor == 1
    assert dftk.model_DFT(LATTICE, [Si, Si], pos, functionals=dftk.LDA()).term_types[0] == "Kinetic"
    m = dftk.model_atomic(LATTICE, [Si, Si], pos, kinetic_blowup=dftk.BlowupAbinit(Ecutsm=0.3))
    assert m.term_types[0].blowup.Ecutsm == 0.3 and m.term_names == ["Kinetic", "AtomicLocal", "AtomicNonlocal",
                                                                      "Ewald", "PspCorrection"]


@pytest.fixture(scope="module")
def al_cold():
    """A displaced two-atom aluminium cell (bct setting of fcc) at Marzari-Vanderbilt smearing, SCF in the oracle."""
    from oracle.basis import Element, Model, PlaneWaveBasis
    from oracle import scf
    a = 7.65339
    lat = np.diag([a / math.sqrt(2), a / math.sqrt(2), a])
    pos = [np.array([0.01, -0.02, 0.015]), np.array([0.5, 0.5, 0.5])]

    def basis_at(p, fft_size=None, ref=None):
        m = Model(lat, [Element("Al")] * 2, p, temperature=0.02, smearing="MarzariVanderbilt", symmetries=False)
        if ref is None:
            return PlaneWaveBasis(m, 5, kgrid=(2, 2, 2))
        return PlaneWaveBasis(m, 5, fft_size=ref.fft_size, kcoords=ref.kcoords_global, kweights=ref.kweights_global)
    with so.extended():
        b = basis_at(pos)
        res = scf.self_consistent_field(b, tol=1e-10, maxiter=80, mixing="kerker")
    assert res["converged"]
    return pos, basis_at, b, res


def test_oracle_cold_smearing_forces_are_free_energy_derivative(al_cold):
    """test/forces.jl:59-88 at Marzari-Vanderbilt smearing: -dF/dx of the free energy (Entropy included) from two
    re-converged oracle SCFs equals the Hellmann-Feynman force, which pins the entropy term end to end."""
    from oracle import scf, forces
    pos, basis_at, b, res = al_cold
    assert abs(res["energies"]["Entropy"]) > 1e-6
    total, _ = forces.compute_forces(b, res["psi"], res["occupation"], res["rho"])
    direction = np.array([0.6, -0.64, 0.48])
    h = 1e-4

    def free_energy(e):
        p = [x.copy() for x in pos]
        p[0] = p[0] + e * direction
        with so.extended():
            r = scf.self_consistent_field(basis_at(p, ref=b), rho=res["rho"], tol=1e-10, maxiter=80, mixing="kerker")
        return r["energies"]["total"]
    fd = -(free_energy(h) - free_energy(-h)) / (2 * h)
    assert np.linalg.norm(total[0]) > 1e-3
    assert abs(float(direction @ total[0]) - fd) < 2e-6
