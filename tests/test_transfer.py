"""CPU checks of the basis transfers: the NumPy restatement (transfer_oracle.py) against the reference's own identities
(test/transfer.jl) and against scipy, and the kernel bodies of transfer_core.cuh under host emulation
(tests/hostemu/emu_transfer.cu) against the restatement."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
from scipy import ndimage

import transfer_oracle as T
from oracle.basis import Element, Kpoint, Model, PlaneWaveBasis, compute_fft_size, index_G_vectors
from oracle.scf import symmetrize_rho
from silicon import LATTICE, POSITIONS

HERE = os.path.dirname(os.path.abspath(__file__))
EPS = np.finfo(float).eps
RECIP = 2 * math.pi * np.linalg.inv(LATTICE.T)


def _kpt(k, fft_size, Ecut):
    return Kpoint(0, k, RECIP, fft_size, Ecut)


def _rand(shape, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _matrix(i, o, n_in, n_out):
    M = np.zeros((n_out, n_in))
    M[o, i] = 1.0
    return M


# ------------------------------------------------------------------ oracle against test/transfer.jl
@pytest.mark.parametrize("k", [(0.25, 0.25, 0.25), (0.0, 0.0, 0.0), (-0.25, 0.25, -0.5)])
def test_blochwave_small_big_small_and_transfer_matrices(k):
    fs, fb = compute_fft_size(LATTICE, 5), compute_fft_size(LATTICE, 10)
    ks, kb = _kpt(k, fs, 5), _kpt(k, fb, 10)
    psi = _rand((ks.n_G, 4), 1)
    psi_b = T.transfer_blochwave_kpt(psi, ks.G_vectors, k, fb, kb.mapping, k)
    psi_bb = T.transfer_blochwave_kpt(psi_b, kb.G_vectors, k, fs, ks.mapping, k)
    assert np.linalg.norm(psi - psi_bb) < EPS
    Tm = _matrix(*T.transfer_mapping_kpt(ks.G_vectors, k, fb, kb.mapping, k), ks.n_G, kb.n_G)
    Tb = _matrix(*T.transfer_mapping_kpt(kb.G_vectors, k, fs, ks.mapping, k), kb.n_G, ks.n_G)
    assert np.abs(Tb @ Tm - np.eye(ks.n_G)).max() < EPS
    P = Tm @ Tb
    np.testing.assert_allclose(P @ P, P)


def test_blochwave_to_equivalent_kpoint_and_back():
    k, dG = np.array([0.25, -0.25, 0.5]), np.array([1, 0, -1])
    fs = compute_fft_size(LATTICE, 8)
    ka, kb = _kpt(k, fs, 8), _kpt(k + dG, fs, 8)
    assert ka.n_G == kb.n_G
    psi = _rand((ka.n_G, 3), 2)
    there = T.transfer_blochwave_kpt(psi, ka.G_vectors, k, fs, kb.mapping, k + dG)
    back = T.transfer_blochwave_kpt(there, kb.G_vectors, k + dG, fs, ka.mapping, k)
    assert np.array_equal(back, psi)
    # the Bloch wave is unchanged: the k+G vectors carrying each coefficient agree
    i, o = T.transfer_mapping_kpt(ka.G_vectors, k, fs, kb.mapping, k + dG)
    np.testing.assert_array_equal(ka.G_vectors[i] + k, kb.G_vectors[o] + k + dG)


def _fft(f, fs):
    return np.fft.fftn(f.reshape(fs[2], fs[1], fs[0])).reshape(-1) / f.size


def _ifft(c, fs):
    return np.real(np.fft.ifftn(c.reshape(fs[2], fs[1], fs[0])).reshape(-1) * c.size)


def _transfer_density(rho, fi, fo):
    return _ifft(T.block_copy(_fft(rho, fi)[None], fi, fo)[0], fo)


def test_density_small_big_small_is_identity():
    fs, fb = (15, 30, 1), (20, 33, 11)
    rng = np.random.default_rng(3)
    c = _fft(rng.random(int(np.prod(fs))), fs)
    from oracle.basis import G_vectors
    Gall = G_vectors(fs)
    c[index_G_vectors(fs, -Gall) < 0] = 0            # enforce_real!
    rho = _ifft(c, fs)
    rho_bb = _transfer_density(_transfer_density(rho, fs, fb), fb, fs)
    np.testing.assert_allclose(rho_bb, rho, rtol=10 * EPS, atol=10 * EPS * np.abs(rho).max())


def test_density_big_small_big_keeps_the_small_components():
    from oracle.basis import G_vectors
    fb, fs = (16, 24, 1), (9, 10, 1)
    rho = np.random.default_rng(4).random(int(np.prod(fb)))
    rho_ss = _transfer_density(_transfer_density(rho, fb, fs), fs, fb)
    d = _fft(rho - rho_ss, fb)
    Gb = G_vectors(fb)
    keep = (index_G_vectors(fs, Gb) >= 0) & (index_G_vectors(fs, -Gb) >= 0)
    assert keep.sum() > 50
    assert np.abs(d[keep]).max() < 10 * EPS


# ------------------------------------------------------------------ apply_symop
def _si_symmetric_basis():
    m = Model(LATTICE, [Element("Si")] * 2, POSITIONS)
    return Model, PlaneWaveBasis(m, 6, fft_size=(18, 18, 18), kcoords=[[0.0, 0.0, 0.0]], kweights=[1.0])


def _density(fs, G, psi, occ):
    N = int(np.prod(fs))
    rho = np.zeros(N)
    lin = index_G_vectors(fs, G)
    for n in range(psi.shape[1]):
        c = np.zeros(N, dtype=complex)
        c[lin] = psi[:, n]
        rho += occ[n] * np.abs(np.fft.ifftn(c.reshape(fs[2], fs[1], fs[0])).reshape(-1) * N) ** 2
    return rho


def test_apply_symop_keeps_norms_and_reproduces_symmetrize_rho():
    _, b = _si_symmetric_basis()
    syms = b.symmetries
    assert len(syms) == 48 and any(np.any(np.abs(s.tau) > 1e-12) for s in syms), "Fd-3m with fractional translations"
    k = np.array([0.25, -0.125, 0.375])
    kp = _kpt(k, b.fft_size, b.Ecut)
    psi = _rand((kp.n_G, 3), 5)
    occ = np.array([2.0, 1.0, 0.5])
    rho = _density(b.fft_size, kp.G_vectors, psi, occ)
    acc = np.zeros_like(rho)
    from oracle.basis import normalize_kpoint_coordinate
    for s in syms:
        Sk = normalize_kpoint_coordinate(s.S @ k)
        ksym = _kpt(Sk, b.fft_size, b.Ecut)
        assert ksym.n_G == kp.n_G
        psi_s = T.apply_symop(s.S, s.tau, k, b.fft_size, kp.G_vectors, psi, ksym.G_vectors)
        np.testing.assert_allclose(np.linalg.norm(psi_s, axis=0), np.linalg.norm(psi, axis=0), rtol=1e-14)
        acc += _density(b.fft_size, ksym.G_vectors, psi_s, occ)
    ref = symmetrize_rho(b, rho[None])[0]
    np.testing.assert_allclose(acc / len(syms), ref, rtol=0, atol=1e-12 * np.abs(ref).max())


# ------------------------------------------------------------------ B-spline
GRIDS = [((12, 12, 12), (18, 18, 18)), ((18, 18, 18), (12, 12, 12)), ((18, 20, 24), (25, 27, 30)),
         ((25, 27, 30), (18, 20, 24)), ((9, 10, 11), (9, 10, 11))]


def _smooth(grid, seed):
    nx, ny, nz = grid
    Z, Y, X = np.meshgrid(np.arange(nz) / nz, np.arange(ny) / ny, np.arange(nx) / nx, indexing="ij")
    rng = np.random.default_rng(seed)
    f = 1.0 + 0.1 * rng.random((nz, ny, nx))
    return f + np.cos(2 * math.pi * (X + 2 * Y)) + 0.5 * np.sin(2 * math.pi * (Z - X))


def _scipy(f, grid_out, rep=(1, 1, 1)):
    nz, ny, nx = f.shape
    nxo, nyo, nzo = grid_out
    Z, Y, X = np.meshgrid(np.arange(nzo), np.arange(nyo), np.arange(nxo), indexing="ij")
    coords = [Z * rep[2] * nz / nzo, Y * rep[1] * ny / nyo, X * rep[0] * nx / nxo]
    return ndimage.map_coordinates(f, coords, order=2, mode="grid-wrap")


@pytest.mark.parametrize("grid_in,grid_out", GRIDS)
def test_bspline_oracle_matches_scipy(grid_in, grid_out):
    f = _smooth(grid_in, 6)
    out = T.interpolate_density(f, grid_out)
    ref = f if grid_in == grid_out else _scipy(f, grid_out)
    np.testing.assert_allclose(out, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())


def test_bspline_supercell_form():
    f = _smooth((9, 10, 8), 7)
    np.testing.assert_array_equal(T.interpolate_density(f, (18, 20, 16), rep=(2, 2, 2)), np.tile(f, (2, 2, 2)))
    out = T.interpolate_density(f, (20, 17, 24), rep=(2, 2, 3))
    ref = _scipy(f, (20, 17, 24), rep=(2, 2, 3))
    np.testing.assert_allclose(out, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())


# ------------------------------------------------------------------ host emulation of the kernel bodies
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu_transfer") / "libemu_transfer.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                           "-o", so, os.path.join(HERE, "hostemu", "emu_transfer.cu")])
    return ctypes.CDLL(so)


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _emu_tables(emu, G, M, delta, tau, lookup, fs):
    n = len(G)
    G = np.ascontiguousarray(G, dtype=np.int64)
    idx = np.empty(n, dtype=np.int64)
    phase = np.empty(n, dtype=np.complex128)
    emu.emu_tr_tables(ctypes.c_int64(n), _p(G), _p(np.ascontiguousarray(M, dtype=np.int32)),
                      _p(np.ascontiguousarray(delta, dtype=np.int32)), _p(np.ascontiguousarray(tau, dtype=np.float64)),
                      _p(lookup), *fs, _p(idx), _p(phase))
    return idx, phase


def _emu_remap(emu, src_rows, idx, phase, n_dst, dst=None, row_offset=0):
    src_rows = np.ascontiguousarray(src_rows)
    if dst is None:
        dst = np.full((src_rows.shape[0], n_dst), np.nan + 0j)
    emu.emu_tr_remap(ctypes.c_int64(src_rows.shape[0]), _p(src_rows), ctypes.c_int64(src_rows.shape[1]), _p(dst),
                     ctypes.c_int64(dst.shape[1]), ctypes.c_int64(row_offset), ctypes.c_int64(n_dst), _p(idx), _p(phase))
    return dst


def _lookup(fs, kp):
    lk = -np.ones(int(np.prod(fs)), dtype=np.int64)
    lk[kp.mapping] = np.arange(kp.n_G)
    return lk


def test_emu_transfer_tables_and_remap_match_oracle(emu):
    k = (0.25, -0.25, 0.5)
    fs, fb = compute_fft_size(LATTICE, 8), compute_fft_size(LATTICE, 12)
    for (f_in, E_in), (f_out, E_out), dG in [((fs, 8), (fb, 12), (0, 0, 0)), ((fb, 12), (fs, 8), (0, 0, 0)),
                                            ((fs, 8), (fs, 8), (1, 0, -1))]:
        ki, ko = _kpt(k, f_in, E_in), _kpt(np.add(k, dG), f_out, E_out)
        psi = _rand((ki.n_G, 5), 8)
        ref = T.transfer_blochwave_kpt(psi, ki.G_vectors, k, f_out, ko.mapping, np.add(k, dG))
        idx, _ = _emu_tables(emu, ko.G_vectors, np.eye(3), dG, np.zeros(3), _lookup(f_in, ki), f_in)
        out = _emu_remap(emu, psi.T, idx, None, ko.n_G)
        assert np.array_equal(out.T, ref)


def test_emu_symop_tables_match_oracle(emu):
    _, b = _si_symmetric_basis()
    k = np.array([0.25, -0.125, 0.375])
    kp = _kpt(k, b.fft_size, b.Ecut)
    psi = _rand((kp.n_G, 2), 9)
    from oracle.basis import normalize_kpoint_coordinate
    n_exact = 0
    for s in b.symmetries:
        Sk_raw = s.S @ k
        Sk = normalize_kpoint_coordinate(Sk_raw)
        ksym = _kpt(Sk, b.fft_size, b.Ecut)
        kshift = np.rint(Sk - Sk_raw).astype(np.int64)
        invS = np.rint(np.linalg.inv(s.S)).astype(np.int32)
        idx, phase = _emu_tables(emu, ksym.G_vectors, invS, kshift, s.tau, _lookup(b.fft_size, kp), b.fft_size)
        # the table: index of S^-1 (G + kshift) in k's sphere, exp(-2 pi i (G + kshift).tau) (exact +-1, +-i here)
        Gf = ksym.G_vectors + kshift
        pos = {tuple(g): i for i, g in enumerate(kp.G_vectors)}
        assert np.array_equal(idx, [pos[tuple(invS @ g)] for g in Gf])
        ref_phase = np.exp(-2j * math.pi * (Gf @ s.tau))
        np.testing.assert_allclose(phase, ref_phase, rtol=0, atol=1e-15)
        if np.all(np.isin(phase.real, (-1.0, 0.0, 1.0))) and np.all(np.isin(phase.imag, (-1.0, 0.0, 1.0))):
            n_exact += 1
        out = _emu_remap(emu, psi.T, idx, phase, ksym.n_G)
        ref = T.apply_symop(s.S, s.tau, k, b.fft_size, kp.G_vectors, psi, ksym.G_vectors)
        np.testing.assert_allclose(out.T, ref, rtol=0, atol=1e-15 * np.abs(ref).max())
    assert n_exact == len(b.symmetries)


def test_emu_remap_row_offset_and_zero_fill(emu):
    src = _rand((3, 7), 10)
    idx = np.array([6, -1, 0, 3, -1], dtype=np.int64)
    dst = np.full((8, 5), 7.0 + 0j)
    _emu_remap(emu, src, idx, None, 5, dst=dst, row_offset=4)
    assert np.array_equal(dst[:4], np.full((4, 5), 7.0 + 0j)) and np.array_equal(dst[7:], np.full((1, 5), 7.0 + 0j))
    ref = np.where(idx >= 0, src[:, np.maximum(idx, 0)], 0)
    assert np.array_equal(dst[4:7], ref)


@pytest.mark.parametrize("fi,fo", [((15, 30, 1), (20, 33, 11)), ((20, 33, 11), (15, 30, 1)), ((16, 24, 1), (9, 10, 1)),
                                   ((9, 10, 4), (16, 24, 5)), ((8, 8, 8), (8, 8, 8))])
def test_emu_block_copy_matches_oracle(emu, fi, fo):
    f = np.ascontiguousarray(_rand((2, int(np.prod(fi))), 11))
    out = np.full((2, int(np.prod(fo))), np.nan + 0j)
    emu.emu_tr_block_copy(_p(f), *fi, _p(out), *fo, ctypes.c_int64(2))
    assert np.array_equal(out, T.block_copy(f, fi, fo))


def test_emu_bspline_matches_oracle(emu):
    for grid_in, grid_out in GRIDS[:4]:
        f = _smooth(grid_in, 12)
        fac = np.empty(f.size)
        emu.emu_tr_prefilter_factor(*grid_in, _p(fac))
        c = np.ascontiguousarray(np.real(np.fft.ifftn(np.fft.fftn(f) * fac.reshape(f.shape))))
        np.testing.assert_allclose(c, T.bspline_coefficients(f), rtol=0, atol=1e-13 * np.abs(c).max())
        out = np.empty(int(np.prod(grid_out)))
        emu.emu_tr_bspline(_p(c), *grid_in, _p(np.ones(3, dtype=np.int32)), _p(out), *grid_out, 0)
        ref = T.interpolate_density(f, grid_out).reshape(-1)
        np.testing.assert_allclose(out, ref, rtol=0, atol=1e-13 * np.abs(ref).max())
    f = np.ascontiguousarray(_smooth((9, 10, 8), 13))
    out = np.empty(18 * 20 * 16)
    emu.emu_tr_bspline(_p(f), 9, 10, 8, _p(np.array([2, 2, 2], dtype=np.int32)), _p(out), 18, 20, 16, 1)
    assert np.array_equal(out, np.tile(f, (2, 2, 2)).reshape(-1))
