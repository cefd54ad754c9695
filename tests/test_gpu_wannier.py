"""GPU tests of the Wannier90 interface (wannier.py over dftk_b200_overlap_multi): the overlaps M^{k,b} and projections A_k
against the literal NumPy restatement (tests/wannier_oracle.py) on both product paths, the Γ-point supercell identity, the
gauge-invariant spread sum through symmetry unfolding, the written files, and run_wannier90 against a stub executable."""
import os

import numpy as np
import pytest

import wannier_oracle as W
from silicon import LATTICE, POSITIONS
from test_wannier import write_stub

pytestmark = pytest.mark.gpu


def _si(dftk, symmetries=True):
    Si = dftk.ElementPsp("Si")
    return dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), symmetries=symmetries)


def _nnkp(basis):
    return W.nnkp_list([k.coordinate for k in basis.kpoints], basis.model.recip_lattice, basis.kgrid.kgrid_size)


def _spread_sum(M, nnkpts, weights_of_pair):
    return sum(w * float(np.sum(np.abs(m) ** 2)) for m, w in zip(M, weights_of_pair))


@pytest.fixture(scope="module")
def shifted_scf():
    """Si LDA on a 3³ grid shifted by ½ (neighbours across the zone boundary have G_shift != 0), 64 bands, unfolded."""
    import dftk_b200 as dftk
    basis = dftk.PlaneWaveBasis(_si(dftk), Ecut=10, kgrid=dftk.MonkhorstPack((3, 3, 3), (0.5, 0.5, 0.5)))
    r = dftk.self_consistent_field(basis, tol=1e-8, nbandsalg=dftk.FixedBands(64))
    return dftk.unfold_bz(r)


@pytest.mark.parametrize("n_bands", [4, 12, 32, 33, 64])
def test_overlaps_match_oracle(shifted_scf, n_bands):
    from dftk_b200.wannier import _mmn_all
    basis, psi = shifted_scf["basis"], shifted_scf["psi"]
    nntot, nnkpts, _, _ = _nnkp(basis)
    assert any(any(g) for _, _, g in nnkpts)
    M = _mmn_all(basis, psi, nnkpts, n_bands)
    G = [k.G_vectors.cpu().numpy() for k in basis.kpoints]
    P = [p.cpu().numpy() for p in psi]
    scale = max(np.abs(M).max(), 1e-300)
    for (ik, ikb, Gs), m in zip(nnkpts, M):
        ref = W.overlap_Mmn_k_kpb(G[ik], P[ik], G[ikb], P[ikb], Gs, n_bands)
        assert np.abs(m - ref).max() <= 1e-12 * scale
    # M^{k,b} = (M^{k+b,-b})^† : the reverse pair is k' = k+b with shift -G_shift
    where = {(ik, ikb, tuple(g)): n for n, (ik, ikb, g) in enumerate(nnkpts)}
    for n, (ik, ikb, Gs) in enumerate(nnkpts):
        back = where[(ikb, ik, tuple(-x for x in Gs))]
        assert np.abs(M[n] - M[back].conj().T).max() <= 1e-13 * scale
    # the single-pair entry point agrees with the batched call
    import dftk_b200 as dftk
    ik, ikb, Gs = nnkpts[5]
    assert np.array_equal(dftk.overlap_Mmn_k_kpb(basis, psi, ik, ikb, Gs, n_bands), M[5])
    # a rerun is bit-identical
    assert np.array_equal(_mmn_all(basis, psi, nnkpts, n_bands), M)


def test_gamma_supercell_identity():
    """At Γ of the supercell every neighbour is a pure G shift: the spread sum S = Σ_{k,b} w_b Σ_{mn} |M^{k,b}_{mn}|² of the
    unit cell's 4 valence bands equals the supercell's, with the supercell's own b-vectors (the same Cartesian vectors)."""
    import dftk_b200 as dftk
    from dftk_b200.wannier import _mmn_all
    basis = dftk.PlaneWaveBasis(_si(dftk, symmetries=False), Ecut=8, kgrid=(3, 3, 3))
    r = dftk.self_consistent_field(basis, tol=1e-10)
    psi = [p[:4].contiguous() for p in r["psi"]]
    nntot, nnkpts, w, cart = _nnkp(basis)
    S_cell = _spread_sum(_mmn_all(basis, psi, nnkpts, 4), nnkpts, [w[n % nntot] for n in range(len(nnkpts))])
    bs = dftk.cell_to_supercell(basis)
    (psi_sc,) = dftk.cell_to_supercell(psi, basis, bs)
    assert psi_sc.shape[0] == 108
    # supercell b-vectors: the unit cell's Cartesian b are reciprocal lattice vectors of the supercell
    recip_sc = bs.model.recip_lattice
    pairs, weights = [], []
    for b, wb in zip(cart, w):
        Gs = np.linalg.solve(recip_sc, b)
        assert np.abs(Gs - np.round(Gs)).max() < 1e-10
        pairs.append((0, 0, tuple(int(x) for x in np.round(Gs))))
        weights.append(wb)
    S_sc = _spread_sum(_mmn_all(bs, [psi_sc], pairs, 108), pairs, weights)
    assert abs(S_sc - S_cell) <= 1e-12 * abs(S_cell)


def test_symmetry_unfolding_spread():
    """S of the 4 valence bands is gauge-invariant: an unfolded symmetry-reduced SCF gives the symmetry-free SCF's value.
    Observed on an H100: 2101.060415055519 against 2101.0604150445192, a relative difference of 5.2e-12 (both SCFs at
    tol 1e-10)."""
    import dftk_b200 as dftk
    from dftk_b200.wannier import _mmn_all
    out = []
    for sym in (True, False):
        basis = dftk.PlaneWaveBasis(_si(dftk, symmetries=sym), Ecut=8, kgrid=dftk.MonkhorstPack((3, 3, 3), (0.5, 0.5, 0.5)))
        r = dftk.unfold_bz(dftk.self_consistent_field(basis, tol=1e-10))
        b = r["basis"]
        nntot, nnkpts, w, _ = _nnkp(b)
        out.append(_spread_sum(_mmn_all(b, r["psi"], nnkpts, 4), nnkpts, [w[n % nntot] for n in range(len(nnkpts))]))
    rel = abs(out[0] - out[1]) / abs(out[1])
    print(f"spread sum: unfolded {out[0]!r}, symmetry-free {out[1]!r}, relative difference {rel:.3e}")
    assert rel < 1e-6


def _projections(dftk):
    projs, refs = [], []
    c = np.array([0.3, -0.2, 0.45])
    projs.append(dftk.GaussianWannierProjection(c))
    refs.append(("g", c))
    for n in (1, 2, 3):
        for l in range(4):
            for m in range(-l, l + 1):
                cc = np.array([0.1 * n, 0.05 * l, -0.07 * m + 0.2])
                projs.append(dftk.HydrogenicWannierProjection(cc, n, l, m, 1.7))
                refs.append(("h", cc, n, l, m, 1.7))
    return projs, refs


def test_projections_match_oracle(shifted_scf):
    import dftk_b200 as dftk
    from dftk_b200.wannier import _amn_all
    basis, psi = shifted_scf["basis"], shifted_scf["psi"]
    projs, refs = _projections(dftk)
    sel = [(8, list(range(30))), (8, list(range(30, len(projs)))), (40, list(range(len(projs))))]   # small and large paths
    for n_bands, ids in sel:
        use = [projs[i] for i in ids]
        A = _amn_all(basis, psi, use, n_bands)
        for ik in (0, 7, len(basis.kpoints) - 1):
            kpt = basis.kpoints[ik]
            ps = basis.Gplusk_vectors(kpt).cpu().numpy()
            recip = basis.model.recip_lattice
            gn = [W.gaussian(ps, recip, refs[i][1]) if refs[i][0] == "g" else W.hydrogenic(ps, recip, *refs[i][1:])
                  for i in ids]
            ref = W.compute_amn_kpoint(psi[ik].cpu().numpy(), gn, n_bands)
            assert np.abs(A[ik] - ref).max() <= 1e-11 * np.abs(ref).max()
            single = dftk.compute_amn_kpoint(basis, kpt, psi[ik], use, n_bands)
            assert np.abs(single - ref).max() <= 1e-11 * np.abs(ref).max()


def _read_complex_block(lines):
    return np.array([complex(float(a), float(b)) for a, b in (l.split()[-2:] for l in lines)])


def test_written_files(tmp_path):
    import dftk_b200 as dftk
    from dftk_b200.wannier import _mmn_all, _amn_all
    basis0 = dftk.PlaneWaveBasis(_si(dftk), Ecut=8, kgrid=dftk.MonkhorstPack((2, 2, 2), (0.5, 0.5, 0.5)))
    scfres = dftk.self_consistent_field(basis0, tol=1e-8, nbandsalg=dftk.FixedBands(8))
    su = dftk.unfold_bz(scfres)
    basis, psi = su["basis"], su["psi"]
    nntot, nnkpts, _, _ = _nnkp(basis)
    prefix = str(tmp_path / "w" / "si")
    projs = [dftk.GaussianWannierProjection(c) for c in np.random.default_rng(1).random((4, 3))]

    def preprocess():
        W.write_nnkp(prefix + ".nnkp", nntot, nnkpts)
        return dftk.read_w90_nnkp(prefix)

    dftk.write_wannier90_files(preprocess, scfres, n_bands=6, n_wannier=4, projections=projs, fileprefix=prefix,
                               wannier_plot=True, num_iter=100)
    n_k = len(basis.kpoints)
    eig = open(prefix + ".eig").read().splitlines()
    vals = np.array([float(l.split()[2]) for l in eig]).reshape(n_k, 6)
    np.testing.assert_allclose(vals, np.array([e[:6] for e in su["eigenvalues"]]) * 27.211386245988, rtol=0, atol=1e-12)
    mmn = open(prefix + ".mmn").read().splitlines()
    assert mmn[1].split() == ["6", str(n_k), str(nntot)]
    M = _mmn_all(basis, psi, nnkpts, 6)
    for n, (ik, ikb, Gs) in enumerate(nnkpts):
        head = mmn[2 + n * 37]
        assert [int(x) for x in head.split()] == [ik + 1, ikb + 1, *Gs]
        vals = _read_complex_block(mmn[3 + n * 37:3 + n * 37 + 36])
        np.testing.assert_allclose(vals, M[n].T.reshape(-1), rtol=0, atol=1e-15)   # %22.18f
    amn = open(prefix + ".amn").read().splitlines()
    A = _amn_all(basis, psi, projs, 6)
    vals = _read_complex_block(amn[2:]).reshape(n_k, 4, 6)
    np.testing.assert_allclose(vals, np.transpose(A, (0, 2, 1)), rtol=0, atol=1e-15)
    assert [int(x) for x in amn[2 + 7].split()[:3]] == [2, 2, 1]
    win = open(prefix + ".win").read()
    assert "wannier_plot   = True" in win and "num_iter" in win
    nx, ny, nz = basis.fft_size
    for ik in (0, n_k - 1):
        lines = open(os.path.join(str(tmp_path / "w"), "UNK%05i.1" % (ik + 1))).read().splitlines()
        assert lines[0].split() == [str(nx), str(ny), str(nz), str(ik + 1), "6"]
        assert len(lines) == 1 + 6 * basis.N
        kpt = basis.kpoints[ik]
        for band in (0, 5):
            ref = W.unk(basis.fft_size, kpt.mapping.cpu().numpy(), psi[ik][band].cpu().numpy(), basis.model.unit_cell_volume)
            for j in (0, 17, basis.N - 1):
                got = complex(*(float(x) for x in lines[1 + band * basis.N + j].split()))
                assert abs(got - ref[j]) <= 1e-15 + 1e-12 * np.abs(ref).max()


def test_spin_polarised_raises(tmp_path):
    import dftk_b200 as dftk
    Fe = dftk.ElementPsp("Fe", functional="pbe")
    lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
    model = dftk.model_DFT(lat, [Fe], [[0, 0, 0]], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0])
    basis = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=(2, 2, 2))
    scfres = dict(basis=basis)
    with pytest.raises(NotImplementedError):
        dftk.write_wannier90_files(lambda: None, scfres, n_bands=4, n_wannier=4, projections=[None] * 4,
                                   fileprefix=str(tmp_path / "x"), wannier_plot=False)


def test_run_wannier90_end_to_end(tmp_path, monkeypatch):
    import dftk_b200 as dftk
    basis0 = dftk.PlaneWaveBasis(_si(dftk), Ecut=8, kgrid=(2, 2, 2))
    scfres = dftk.self_consistent_field(basis0, tol=1e-8)
    bu = dftk.unfold_bz(basis0)
    nntot, nnkpts, _, _ = _nnkp(bu)
    ref = tmp_path / "ref.nnkp"
    W.write_nnkp(str(ref), nntot, nnkpts)
    bindir = tmp_path / "bin"
    bindir.mkdir()
    log = str(tmp_path / "calls.log")
    write_stub(str(bindir), ref.read_text(), log)
    monkeypatch.setenv("PATH", str(bindir) + os.pathsep + os.environ.get("PATH", ""))
    monkeypatch.delenv("WANNIER90", raising=False)
    prefix = str(tmp_path / "wannier90" / "si")
    assert dftk.run_wannier90(scfres, n_bands=4, fileprefix=prefix) == prefix
    d = str(tmp_path / "wannier90")
    assert open(log).read().splitlines() == [d + " -pp si", d + " si"]
    for ext in (".win", ".nnkp", ".eig", ".amn", ".mmn", ".wout"):
        assert os.path.isfile(prefix + ext), ext
    mmn = open(prefix + ".mmn").read().splitlines()
    assert mmn[1].split() == ["4", str(len(bu.kpoints)), str(nntot)]
