"""Self-check of tests/fft_reference.py: the direct DFT against numpy.fft, the stage forms against the oracle's ifft_kpt /
fft_kpt, and the shape of the generated spheres."""
import numpy as np
import pytest

import fft_reference as fr


@pytest.mark.parametrize("shape", [(8, 9, 10), (15, 18, 25), (7, 11, 13), (1, 4, 25), (97, 2, 3), (256, 3, 5)])
def test_direct_dft_matches_numpy_fft(shape):
    nx, ny, nz = shape
    rng = np.random.default_rng(sum(shape))
    x = rng.standard_normal((2, nz, ny, nx)) + 1j * rng.standard_normal((2, nz, ny, nx))
    fwd = fr.dft3(x.reshape(2, -1), shape, -1).reshape(x.shape)
    bwd = fr.dft3(x.reshape(2, -1), shape, +1).reshape(x.shape)
    ref_f = np.fft.fftn(x, axes=(1, 2, 3))
    ref_b = np.fft.ifftn(x, axes=(1, 2, 3)) * (nx * ny * nz)
    assert np.abs(fwd - ref_f).max() <= 1e-14 * np.abs(ref_f).max()
    assert np.abs(bwd - ref_b).max() <= 1e-14 * np.abs(ref_b).max()


def test_dft_matrix_phases_are_exact():
    """Entries of a long axis are the correctly rounded cos / sin of the reduced phase (no drift with j m)."""
    n = 512
    M = fr.dft_matrix(n, -1)
    j, m = 511, 509
    ang = 2 * np.pi * ((j * m) % n) / n
    assert abs(M[j, m] - np.exp(-1j * ang)) <= 2e-16
    np.testing.assert_array_equal(M, M.T)
    assert np.abs(M @ fr.dft_matrix(n, +1) - n * np.eye(n)).max() < 1e-11


def test_stage_forms_match_oracle_conventions():
    """The four reference stage forms against oracle/basis.py ifft_kpt / fft_kpt on a silicon k-point."""
    from oracle.basis import Element, Model, PlaneWaveBasis
    from silicon import LATTICE, POSITIONS
    m = Model(LATTICE, [Element("Si")] * 2, POSITIONS, symmetries=False)
    b = PlaneWaveBasis(m, 6, fft_size=(15, 16, 18), kcoords=[[0.1, -0.2, 0.3]], kweights=[1.0])
    kpt, shape = b.kpoints[0], b.fft_size
    mp = np.asarray(kpt.mapping, dtype=np.int64)
    rng = np.random.default_rng(4)
    psi = rng.standard_normal((2, kpt.n_G)) + 1j * rng.standard_normal((2, kpt.n_G))
    V = rng.standard_normal(b.N)
    kin = rng.random(kpt.n_G)
    f = rng.standard_normal((2, b.N)) + 1j * rng.standard_normal((2, b.N))
    w = np.array([0.7, 1.3])
    ref_apply = np.stack([b.fft_kpt(kpt, b.ifft_kpt(kpt, p, False) * V / b.N, False) + kin * p for p in psi])
    ref_cube = np.stack([b.ifft_kpt(kpt, p) for p in psi])
    ref_back = np.stack([b.fft_kpt(kpt, x) for x in f])
    ref_rho = sum(w[i] * b.ifft_normalization ** 2 * np.abs(b.ifft_kpt(kpt, psi[i], False)) ** 2 for i in range(2))
    for got, ref in ((fr.local_apply(psi, mp, shape, V, kin), ref_apply),
                     (fr.sphere_to_real(psi, mp, shape, b.ifft_normalization), ref_cube),
                     (fr.real_to_sphere(f, mp, shape, b.fft_normalization), ref_back),
                     (fr.density(psi, w, mp, shape, b.ifft_normalization), ref_rho)):
        assert np.abs(got - ref).max() <= 1e-14 * np.abs(ref).max()


def test_reg_pairs_parsed_from_the_plan_header():
    pairs = fr.reg_pairs()
    lengths = {a * b for a, b in pairs}
    assert {15, 150, 192, 256} <= lengths and len(pairs) >= 30
    assert all(2 <= a <= 16 and 2 <= b <= 25 for a, b in pairs)


@pytest.mark.parametrize("shape", [(15, 18, 25), (256, 18, 25), (25, 16, 18), (18, 25, 97)])
def test_ellipsoid_mapping(shape):
    nx, ny, nz = shape
    N = nx * ny * nz
    full = fr.ellipsoid_mapping(shape, fr.FULL)
    np.testing.assert_array_equal(full, np.arange(N))
    half = fr.ellipsoid_mapping(shape, fr.HALF)
    assert np.all(np.diff(half) > 0) and 0.03 * N < half.size < 0.1 * N
    # asymmetric: the mirror image -G of the set is a different set
    cz, cy, cx = np.unravel_index(half, (nz, ny, nx))
    g = [fr.centred_freqs(n)[c] for n, c in ((nx, cx), (ny, cy), (nz, cz))]
    mirror = np.sort(np.ravel_multi_index(tuple((-gi) % n for gi, n in zip(g[::-1], (nz, ny, nx))), (nz, ny, nx)))
    assert not np.array_equal(mirror, half)
    # it wraps: along each axis the occupied indices form two runs (the range form of the register engine)
    for c, n in ((cx, nx), (cy, ny), (cz, nz)):
        present = np.zeros(n, dtype=bool)
        present[c] = True
        assert fr.index_runs(present) == 2
    np.testing.assert_array_equal(fr.ellipsoid_mapping(shape, 0), [0])
