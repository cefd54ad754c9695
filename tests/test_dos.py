"""Host logic of the densities of states (dftk_b200.dos) against the restatement of dos.jl in tests/dos_oracle.py: the
weights of every smearing (Methfessel-Paxton and Marzari-Vanderbilt give signed ones), the DOS, the PDOS product,
sum_pdos, the zero-temperature errors, and the dispatch of the LdosMixing call form of compute_ldos to its own code."""
from types import SimpleNamespace

import numpy as np
import pytest

import dos_oracle as oracle

KINDS = ["FermiDirac", "Gaussian", "MarzariVanderbilt", ("MethfesselPaxton", 1), ("MethfesselPaxton", 2),
         ("MethfesselPaxton", 3)]


def _basis(n_spin=2, smearing="Gaussian", temperature=0.01, seed=0):
    """A stand-in with what the host logic reads: three k-points per spin, ragged band counts."""
    from dftk_b200.parallel import KpointComm
    rng = np.random.default_rng(seed)
    kw = [0.5, 0.3, 0.2] * n_spin
    spins = [s for s in range(n_spin) for _ in range(3)]
    eig = [np.sort(rng.uniform(-0.3, 0.6, nb)) for nb in [7, 8, 6] * n_spin]
    model = SimpleNamespace(smearing=smearing, temperature=temperature, filled_occupation=2 // n_spin,
                            n_spin_components=n_spin, positions=[np.zeros(3), np.full(3, 0.25)])
    basis = SimpleNamespace(model=model, kweights=kw, kpoints=[SimpleNamespace(spin=s) for s in spins],
                            comm_kpts=KpointComm())
    return basis, eig


@pytest.mark.parametrize("kind", KINDS, ids=str)
def test_weights_match_oracle(kind):
    from dftk_b200 import dos
    basis, eig = _basis(smearing=kind)
    εs = np.linspace(-0.4, 0.7, 37)
    W = dos.dos_weights(basis, eig, εs, kind, 0.01)
    signs = set()
    for w, e in zip(W, eig):
        assert w.shape == (len(εs), len(e))
        ref = np.array([[oracle.ldos_weight(x, ε, 1, kind, 0.01) for x in e] for ε in εs])
        np.testing.assert_allclose(w, ref, rtol=1e-13, atol=1e-13 * np.abs(ref).max())
        signs |= set(np.sign(ref[np.abs(ref) > 1e-8]).tolist())
    # Fermi-Dirac and Gaussian weights are positive; MV and MP are signed
    assert signs == ({1.0} if kind in ("FermiDirac", "Gaussian") else {-1.0, 1.0})


@pytest.mark.parametrize("kind", KINDS, ids=str)
@pytest.mark.parametrize("n_spin", [1, 2])
def test_dos_matches_oracle(kind, n_spin):
    from dftk_b200 import compute_dos
    basis, eig = _basis(n_spin, kind)
    spins = [k.spin for k in basis.kpoints]
    filled = basis.model.filled_occupation
    εs = np.linspace(-0.4, 0.7, 23)
    D = compute_dos(εs, basis, eig)
    assert D.shape == (len(εs), n_spin)
    ref = np.stack([oracle.compute_dos(ε, spins, basis.kweights, eig, n_spin, filled, kind, 0.01) for ε in εs])
    np.testing.assert_allclose(D, ref, rtol=1e-13, atol=1e-13 * np.abs(ref).max())
    d0 = compute_dos(0.1, basis, eig)                         # a number gives (n_spin,)
    assert d0.shape == (n_spin,)
    np.testing.assert_allclose(d0, oracle.compute_dos(0.1, spins, basis.kweights, eig, n_spin, filled, kind, 0.01), rtol=1e-13)
    res = dict(basis=basis, eigenvalues=eig, eF=0.1)           # scfres form, ε = εF by default
    np.testing.assert_array_equal(compute_dos(res), d0)
    np.testing.assert_array_equal(compute_dos(res, εs), D)
    np.testing.assert_allclose(compute_dos(0.1, basis, eig, smearing="FermiDirac", temperature=0.02),
                               oracle.compute_dos(0.1, spins, basis.kweights, eig, n_spin, filled, "FermiDirac", 0.02), rtol=1e-13)


@pytest.mark.parametrize("kind", ["Gaussian", ("MethfesselPaxton", 2)], ids=str)
def test_pdos_matches_oracle(kind, monkeypatch):
    from dftk_b200 import compute_pdos, hubbard
    basis, eig = _basis(2, kind)
    rng = np.random.default_rng(7)
    proj = [rng.random((len(e), 5)) for e in eig]
    labels = [dict(iatom=i // 4, species="X", n=1, l=int(i % 4 > 0), m=0, label="s" if i % 4 == 0 else "p")
              for i in range(5)]
    monkeypatch.setattr(hubbard, "atomic_orbital_projections", lambda b, psi: (proj, labels))
    εs = np.linspace(-0.4, 0.7, 11)
    res = compute_pdos(εs, basis, [None] * len(eig), eig)
    ref = oracle.compute_pdos(εs, [k.spin for k in basis.kpoints], basis.kweights, eig, proj, 2, 1, kind, 0.01)
    assert res.pdos.shape == (len(εs), 5, 2) and res.projector_labels is labels
    np.testing.assert_allclose(res.pdos, ref, rtol=1e-13, atol=1e-13 * np.abs(ref).max())
    pdos, lab, e2 = compute_pdos(εs, basis, [None] * len(eig), eig, positions=basis.model.positions)
    np.testing.assert_array_equal(pdos, res.pdos)
    with pytest.raises(NotImplementedError):
        compute_pdos(εs, basis, [None] * len(eig), eig, positions=[np.zeros(3), np.full(3, 0.2)])


def test_sum_pdos_matches_oracle():
    from dftk_b200 import sum_pdos, PdosResult
    rng = np.random.default_rng(3)
    labels = [dict(iatom=a, species="Si", n=1, l=l, m=m, label="3S" if l == 0 else "3P")
              for a in range(2) for l in range(2) for m in range(-l, l + 1)]
    pdos = rng.random((9, len(labels), 2))
    res = PdosResult(pdos, labels, np.linspace(0, 1, 9))
    for filters in ([lambda o: o["iatom"] == 0], [lambda o: o["l"] == 1], [lambda o: o["label"] == "3S", lambda o: o["iatom"] == 1],
                    [lambda o: False]):
        np.testing.assert_allclose(sum_pdos(res, filters), oracle.sum_pdos(pdos, labels, 9, filters), rtol=1e-14)
    np.testing.assert_allclose(sum_pdos(res, [lambda o: True]), pdos.sum(axis=1), rtol=1e-14)


@pytest.mark.parametrize("what", ["dos", "ldos", "pdos"])
def test_zero_temperature_raises(what):
    from dftk_b200 import compute_dos, compute_ldos, compute_pdos
    basis, eig = _basis(1, "Gaussian", temperature=0.0)
    call = {"dos": lambda **kw: compute_dos(0.1, basis, eig, **kw),
            "ldos": lambda **kw: compute_ldos(np.array([0.1, 0.2]), basis, eig, [None] * 3, **kw),
            "pdos": lambda **kw: compute_pdos([0.1], basis, [None] * 3, eig, **kw)}[what]
    with pytest.raises(ValueError, match="finite temperature"):
        call()
    with pytest.raises(ValueError, match="finite temperature"):
        call(smearing="None", temperature=0.01)
    with pytest.raises(ValueError, match="finite temperature"):
        getattr(oracle, "compute_dos")(0.1, [0], [1.0], [eig[0]], 1, 2, "None", 0.01)


def test_old_ldos_call_form_dispatches_to_old_code(monkeypatch):
    """compute_ldos(basis, eF, eigenvalues, psi, *, temperature) is the LdosMixing form: it reaches scf.compute_ldos with
    the same arguments, and LdosMixing itself keeps calling scf.compute_ldos."""
    import dftk_b200
    from dftk_b200 import scf
    from dftk_b200.basis import PlaneWaveBasis
    calls = []
    monkeypatch.setattr(scf, "compute_ldos", lambda *a, **kw: calls.append((a, kw)) or "old")
    basis = object.__new__(PlaneWaveBasis)
    assert dftk_b200.compute_ldos(basis, 0.25, ["eig"], ["psi"], temperature=0.03) == "old"
    assert calls == [((basis, 0.25, ["eig"], ["psi"]), dict(temperature=0.03, weight_threshold=np.finfo(float).eps))]
    assert dftk_b200.compute_ldos(basis, 0.25, ["eig"], ["psi"], temperature=0.03, weight_threshold=1e-9) == "old"
    assert calls[-1][1] == dict(temperature=0.03, weight_threshold=1e-9)
    assert "compute_ldos(basis, eF, eigenvalues, psi, temperature=Tm)" in open(scf.__file__).read()
