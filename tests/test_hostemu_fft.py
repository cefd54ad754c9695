"""Index-logic test of the FFT pipeline kernel bodies, executed on the host (tests/hostemu/emu.cu
compiles the same __host__ __device__ stage functions the CUDA kernels run).  Checker: the oracle."""
import ctypes
import os
import subprocess
import numpy as np
import pytest

import fft_reference as fr
from oracle.basis import Element, Model, PlaneWaveBasis
from silicon import LATTICE, POSITIONS

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "hostemu", "libhostemu.so")


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "hostemu", "emu.cu")
    csrc = os.path.join(HERE, "..", "dftk.jl_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("fft_core.cuh", "fft_plan.h", "fft_reg.cuh", "fft_radix_gen.cuh", "xc_core.cuh", "forces_core.cuh", "lobpcg_small.cuh", "i8emu_core.cuh", "fft_reg_fwd.cuh")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                               "-Wno-deprecated-gpu-targets", "-o", SO, src])
    return ctypes.CDLL(SO)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _basis(fft_size, Ecut, k):
    m = Model(LATTICE, [Element("Si")] * 2, POSITIONS, symmetries=False)
    return PlaneWaveBasis(m, Ecut, fft_size=fft_size, kcoords=[k], kweights=[1.0])


@pytest.mark.parametrize("fft_size,Ecut,prefix", [((15, 15, 15), 5, "emu"), ((12, 15, 18), 4, "emu"),
                                                  ((17, 20, 21), 6, "emu"), ((27, 27, 27), 15, "emu"),
                                                  ((24, 24, 24), 9, "emu"),
                                                  # register two-pass engine (fft_reg.cuh)
                                                  ((15, 18, 24), 5, "emur"), ((27, 27, 27), 15, "emur"),
                                                  ((24, 16, 20), 6, "emur"), ((20, 27, 15), 5, "emur")])
def test_emulated_pipeline(emu, fft_size, Ecut, prefix):
    lib = emu

    class _E:
        def __getattr__(self, name):
            return getattr(lib, name.replace("emu_", prefix + "_"))
    emu = _E()
    b = _basis(fft_size, Ecut, [0.1, -0.2, 0.3])
    kpt = b.kpoints[0]
    nx, ny, nz = fft_size
    rng = np.random.default_rng(1)
    nb = 3
    npw = ctypes.c_int64(kpt.n_G)
    psi = rng.standard_normal((nb, kpt.n_G)) + 1j * rng.standard_normal((nb, kpt.n_G))
    V = rng.standard_normal(b.N)
    kin = rng.random(kpt.n_G)
    mapping = np.ascontiguousarray(kpt.mapping, dtype=np.int64)
    Vs = np.ascontiguousarray(V / b.N)
    # H psi local + kinetic
    out = np.zeros_like(psi)
    assert emu.emu_apply_local(nx, ny, nz, npw, _p(mapping), _p(psi), nb, _p(Vs), _p(kin), _p(out)) == 0
    ref = np.stack([b.fft_kpt(kpt, b.ifft_kpt(kpt, psi[i], False) * V / b.N, False) + kin * psi[i]
                    for i in range(nb)])
    np.testing.assert_allclose(out, ref, atol=1e-11 * np.abs(ref).max())
    # sphere -> real
    cube = np.zeros((nb, b.N), dtype=complex)
    emu.emu_sphere_to_real(nx, ny, nz, npw, _p(mapping), _p(psi), nb,
                           ctypes.c_double(b.ifft_normalization), _p(cube))
    refc = np.stack([b.ifft_kpt(kpt, psi[i]) for i in range(nb)])
    np.testing.assert_allclose(cube, refc, atol=1e-12 * np.abs(refc).max())
    # real -> sphere
    f = rng.standard_normal((nb, b.N)) + 1j * rng.standard_normal((nb, b.N))
    back = np.zeros_like(psi)
    emu.emu_real_to_sphere(nx, ny, nz, npw, _p(mapping), _p(f), nb,
                           ctypes.c_double(b.fft_normalization), _p(back))
    refb = np.stack([b.fft_kpt(kpt, f[i]) for i in range(nb)])
    np.testing.assert_allclose(back, refb, atol=1e-12 * np.abs(refb).max())
    # density
    w = rng.random(nb)
    rho = np.zeros(b.N)
    emu.emu_density(nx, ny, nz, npw, _p(mapping), _p(psi), nb, _p(w), _p(rho))
    refr = sum(w[i] * np.abs(b.ifft_kpt(kpt, psi[i], False)) ** 2 for i in range(nb))
    np.testing.assert_allclose(rho, refr, atol=1e-11 * refr.max())
    if prefix == "emur":
        assert lib.emur_ranges_ok(nx, ny, nz, npw, _p(mapping)) == 1      # a k-point sphere always has the range form
    # unsorted mapping (construct_from_equivalent_kpt, src/Kpoint.jl:44-56)
    perm = rng.permutation(kpt.n_G)
    out2 = np.zeros_like(psi)
    rc = emu.emu_apply_local(nx, ny, nz, npw, _p(np.ascontiguousarray(mapping[perm])),
                             _p(np.ascontiguousarray(psi[:, perm])), nb, _p(Vs),
                             _p(np.ascontiguousarray(kin[perm])), _p(out2))
    if prefix == "emur":
        assert rc == -9       # register engine needs ascending mappings; such k-blocks use the generic engine
    else:
        assert rc == 0
        np.testing.assert_allclose(out2, ref[:, perm], atol=1e-11 * np.abs(ref).max())


@pytest.mark.parametrize("frac", [fr.HALF, fr.FULL], ids=["half", "full"])
@pytest.mark.parametrize("axis", ["x", "y", "z"])
@pytest.mark.parametrize("n", [a * b for a, b in fr.reg_pairs()])
def test_emulated_register_engine_every_pair(emu, n, axis, frac):
    """Every factor pair of the register engine, on each axis of an (n, 18, 25)-type box, against the direct DFT: local
    apply, sphere -> real, real -> sphere and density, on an off-centre ellipsoid filling half or all of the box."""
    shape = fr.placements(n)[axis]
    nx, ny, nz = shape
    N = nx * ny * nz
    mapping = fr.ellipsoid_mapping(shape, frac)
    assert frac != fr.FULL or mapping.size == N
    npw = ctypes.c_int64(mapping.size)
    assert emu.emur_ranges_ok(nx, ny, nz, npw, _p(mapping)) == 1
    rng = np.random.default_rng(n)
    nb = 2
    psi = rng.standard_normal((nb, mapping.size)) + 1j * rng.standard_normal((nb, mapping.size))
    V = rng.standard_normal(N)
    kin = rng.random(mapping.size)
    ifft_norm, fft_norm = 0.37, 1.9 / N

    def check(got, ref):
        assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()
    out = np.full_like(psi, np.nan)
    assert emu.emur_apply_local(nx, ny, nz, npw, _p(mapping), _p(psi), nb, _p(np.ascontiguousarray(V / N)), _p(kin),
                                _p(out)) == 0
    check(out, fr.local_apply(psi, mapping, shape, V, kin))
    cube = np.full((nb, N), np.nan + 0j)
    assert emu.emur_sphere_to_real(nx, ny, nz, npw, _p(mapping), _p(psi), nb, ctypes.c_double(ifft_norm), _p(cube)) == 0
    check(cube, fr.sphere_to_real(psi, mapping, shape, ifft_norm))
    f = rng.standard_normal((nb, N)) + 1j * rng.standard_normal((nb, N))
    back = np.full_like(psi, np.nan)
    assert emu.emur_real_to_sphere(nx, ny, nz, npw, _p(mapping), _p(f), nb, ctypes.c_double(fft_norm), _p(back)) == 0
    check(back, fr.real_to_sphere(f, mapping, shape, fft_norm))
    w = np.array([1.5, 0.0])
    rho0 = rng.random(N)
    rho = rho0.copy()
    assert emu.emur_density(nx, ny, nz, npw, _p(mapping), _p(psi), nb, _p(w), _p(rho)) == 0
    check(rho - rho0, fr.density(psi, w, mapping, shape))


@pytest.mark.parametrize("fft_size", [(8, 9, 10), (15, 15, 15), (33, 5, 7), (40, 3, 16), (1, 4, 25)])
def test_emulated_cube_fft(emu, fft_size):
    nx, ny, nz = fft_size
    rng = np.random.default_rng(2)
    x = rng.standard_normal((2, nz, ny, nx)) + 1j * rng.standard_normal((2, nz, ny, nx))
    for sign in (-1, 1):
        d = x.copy()
        emu.emu_fft_cube(nx, ny, nz, _p(d), sign, 2)
        ref = np.fft.fftn(x, axes=(1, 2, 3)) if sign < 0 else np.fft.ifftn(x, axes=(1, 2, 3)) * (nx * ny * nz)
        np.testing.assert_allclose(d, ref, atol=1e-12 * np.abs(ref).max())


XC_MASK = {"lda_x": 1, "lda_c_vwn": 2, "lda_c_pw": 4, "gga_x_pbe": 8, "gga_c_pbe": 16}


@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("funs", [("lda_x", "lda_c_vwn"), ("lda_x", "lda_c_pw"), ("gga_x_pbe", "gga_c_pbe")])
def test_emulated_xc_matches_oracle(emu, n_spin, funs):
    """xc_core.cuh (dual-number CUDA functionals, run on the host) against the oracle's XC restatement."""
    from oracle import xc as oxc
    rng = np.random.default_rng(5)
    N = 200
    rho = rng.random((n_spin, N)) * 0.4 + 1e-5
    rho[:, :3] = 0.0                                   # below the density threshold
    rho[:, 3] = 1e-9
    gga = any(f.startswith("gga") for f in funs)
    nsig = (1 if n_spin == 1 else 3) if gga else 0
    sigma = rng.random((max(nsig, 1), N)) * 0.02
    if nsig == 3:
        sigma[1] = np.sqrt(sigma[0] * sigma[2]) * rng.uniform(-1, 1, N)
    e, vr, vs = np.zeros(N), np.zeros((n_spin, N)), np.zeros((max(nsig, 1), N))
    mask = sum(XC_MASK[f] for f in funs)
    assert emu.emu_xc(mask, n_spin, int(gga), ctypes.c_int64(N), _p(rho), _p(sigma), _p(e), _p(vr), _p(vs)) == 0
    ref = oxc.evaluate(list(funs), rho, sigma[:nsig] if gga else None)
    np.testing.assert_allclose(e, ref["e"], rtol=1e-13, atol=1e-16)
    np.testing.assert_allclose(vr, ref["Vrho"], rtol=1e-12, atol=1e-14)
    if gga:
        np.testing.assert_allclose(vs[:nsig], ref["Vsigma"], rtol=1e-11, atol=1e-13)


def test_emulated_symmetrize_matches_oracle(emu):
    """symmetrize_point (accumulate_over_symmetries!, src/symmetry.jl:282-327) against the oracle on silicon."""
    from oracle.scf import symmetrize_rho
    m = Model(LATTICE, [Element("Si")] * 2, POSITIONS)
    b = PlaneWaveBasis(m, 5, fft_size=(12, 12, 12), kcoords=[[0, 0, 0]], kweights=[1.0])
    assert len(b.symmetries) == 48
    rng = np.random.default_rng(9)
    rho = rng.random((1, b.N))
    ref = symmetrize_rho(b, rho)[0]
    rf = np.ascontiguousarray(b.fft_cube(rho[0]))
    invS = np.ascontiguousarray(np.stack([np.rint(np.linalg.inv(s.S)).astype(np.int32) for s in b.symmetries]))
    tau = np.ascontiguousarray(np.stack([s.tau for s in b.symmetries]))
    out = np.zeros_like(rf)
    nx, ny, nz = b.fft_size
    assert emu.emu_symmetrize(nx, ny, nz, _p(rf), _p(out), len(b.symmetries), _p(invS), _p(tau)) == 0
    np.testing.assert_allclose(b.irfft_cube(out), ref, atol=1e-13)


def test_emulated_force_bodies_match_oracle(emu):
    """forces_core.cuh (local-potential forces; the four-projection form of the nonlocal forces) against the oracle's
    restatement of local.jl:152-181 / nonlocal.jl:49-100 on a rattled silicon cell."""
    import math
    from oracle import forces as oforces
    from oracle.psp_hgh import PspHgh
    from oracle.terms import build_projection_vectors
    si = Element("Si", PspHgh.from_table("Si", "lda"))
    pos = [POSITIONS[0] + np.array([0.011, -0.007, 0.004]), POSITIONS[1] + np.array([-0.003, 0.009, 0.006])]
    m = Model(LATTICE, [si, si], pos, symmetries=False)
    b = PlaneWaveBasis(m, 5, fft_size=(15, 16, 18), kcoords=[[0.1, -0.2, 0.3], [0.0, 0.25, 0.5]], kweights=[0.4, 0.6])
    rng = np.random.default_rng(11)
    nx, ny, nz = b.fft_size
    # local
    rho = rng.random((1, b.N)) + 0.1
    ref = np.array(oforces.forces_local(b, rho))
    pn = np.sqrt(np.sum(b.G_cart ** 2, axis=1))
    w = np.ascontiguousarray(np.conj(b.fft_cube(rho[0])) * si.psp.eval_local_fourier(pn) / math.sqrt(m.unit_cell_volume))
    out = np.zeros((2, 3))
    assert emu.emu_local_forces(nx, ny, nz, _p(w), 2, _p(np.ascontiguousarray(np.array(pos))), _p(out)) == 0
    np.testing.assert_allclose(out, ref, rtol=1e-11, atol=1e-12)
    # nonlocal
    nb = 5
    psi = [rng.standard_normal((k.n_G, nb)) + 1j * rng.standard_normal((k.n_G, nb)) for k in b.kpoints]
    occ = [rng.random(nb) * 2 for _ in b.kpoints]
    refn = np.array(oforces.forces_nonlocal(b, psi, occ))
    F = np.zeros((2, 3))
    for ik, kpt in enumerate(b.kpoints):
        P, D = build_projection_vectors(b, kpt)
        n_proj = P.shape[1]
        gpk = np.ascontiguousarray((kpt.G_vectors + kpt.coordinate).T.astype(float))        # (3, n_G)
        psik = np.ascontiguousarray(psi[ik].T)                                              # (nb, n_G) = column-major n_G x nb
        scaled = np.zeros((3 * nb, kpt.n_G), dtype=complex)
        assert emu.emu_scale_by_momentum(ctypes.c_int64(kpt.n_G), ctypes.c_int64(nb), _p(gpk), _p(psik), _p(scaled)) == 0
        np.testing.assert_array_equal(scaled.reshape(3, nb, -1), gpk[:, None, :] * psik[None])
        proj = P.conj().T @ psi[ik]                                                         # (n_proj, nb)
        dproj = np.ascontiguousarray((D @ proj).T)                                          # column-major n_proj x nb
        pa = np.ascontiguousarray((P.conj().T @ scaled.T).T)                                # column-major n_proj x 3 nb
        rows = np.zeros((3, n_proj))
        wts = np.ascontiguousarray(occ[ik] * b.kweights[ik])
        assert emu.emu_nonlocal_force_rows(ctypes.c_int64(n_proj), ctypes.c_int64(nb), _p(dproj), _p(pa), _p(wts), _p(rows)) == 0
        per_atom = n_proj // 2
        for ia in range(2):
            F[ia] += rows[:, ia * per_atom:(ia + 1) * per_atom].sum(axis=1)
    np.testing.assert_allclose(F, refn, rtol=1e-11, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------------
# fused small-matrix LOBPCG bodies (lobpcg_small.cuh): block-list Gram / update products, X*invR, safe_cholesky
# ---------------------------------------------------------------------------------------------------------------
def _lists(blocks):
    """ctypes views of a list of column-major blocks given as (n_cols, n_rows) C-contiguous complex arrays."""
    n = len(blocks)
    ptrs = (ctypes.c_void_p * 3)(*[b.ctypes.data for b in blocks] + [None] * (3 - n))
    lds = (ctypes.c_int64 * 3)(*[b.shape[1] for b in blocks] + [0] * (3 - n))
    cols = (ctypes.c_int * 3)(*[b.shape[0] for b in blocks] + [0] * (3 - n))
    return n, ptrs, lds, cols


def _normest(M):
    d = np.diag(M)
    return np.max(np.abs(d)) + np.linalg.norm(M - np.diag(d))


@pytest.mark.parametrize("rows,cols_a,cols_b", [(2114, (7, 7, 5), (7, 7, 5)), (333, (12,), (12, 3)), (21, (7,), (7,)),
                                                (5442, (15, 15, 15), (15, 15, 15))])
def test_emulated_small_gram_and_updates(emu, rows, cols_a, cols_b):
    rng = np.random.default_rng(5)
    mk = lambda c: np.ascontiguousarray(rng.standard_normal((c, rows)) + 1j * rng.standard_normal((c, rows)))
    A, B = [mk(c) for c in cols_a], [mk(c) for c in cols_b]
    ta, tb = sum(cols_a), sum(cols_b)
    Afull, Bfull = np.concatenate(A, axis=0).T, np.concatenate(B, axis=0).T          # rows x cols
    ref = Afull.conj().T @ Bfull
    for upper in (0, 1):
        C = np.full((tb, ta + 2), np.nan + 0j)                                            # column-major ta(+2 pad) x tb
        for rpc in (64, 128):
            assert emu.emu_small_gram(*_lists(A), *_lists(B), ctypes.c_int64(rows), ctypes.c_int64(rpc), upper, _p(C),
                                      ctypes.c_int64(ta + 2)) == 0
            got = C[:, :ta].T
            sa = np.repeat(np.arange(len(cols_a)), cols_a)
            sb = np.repeat(np.arange(len(cols_b)), cols_b)
            keep = (sb[None, :] >= sa[:, None]) if upper else np.ones((ta, tb), dtype=bool)
            np.testing.assert_allclose(got[keep], ref[keep], rtol=1e-12, atol=1e-11)
            assert upper == 0 or np.all(np.isnan(got[~keep]))                             # skipped blocks stay untouched
    # out = alpha * [A blocks] cm + beta * out
    # (the column counts cover the 8-wide register chunk, the 16-wide one, a 16 + 8 split and the 32-column maximum)
    for ncols in (min(7, ta), 1, 8, 9, 15, 16, 20, 32):
        cm = np.ascontiguousarray(rng.standard_normal((ncols, ta + 1)) + 1j * rng.standard_normal((ncols, ta + 1)))
        out0 = np.ascontiguousarray(rng.standard_normal((ncols, rows)) + 1j * rng.standard_normal((ncols, rows)))
        for alpha, beta in ((1.0, 0.0), (-1.0, 1.0)):
            out = out0.copy()
            assert emu.emu_small_blocks_times(*_lists(A), _p(cm), ta + 1, ncols, _p(out), ctypes.c_int64(rows),
                                              ctypes.c_int64(rows), ctypes.c_double(alpha), ctypes.c_double(beta)) == 0
            want = alpha * (Afull @ cm[:, :ta].T) + beta * out0.T
            np.testing.assert_allclose(out.T, want, rtol=1e-12, atol=1e-11)


@pytest.mark.parametrize("n", [1, 7, 15, 32])
def test_emulated_small_cholesky_qr(emu, n):
    """k_small_chol + k_small_rmul = one pass of ortho! (lobpcg_hyper_impl.jl:216-261): X invR is orthonormal, the
    statistics are those of safe_cholesky / normest (:190-212)."""
    rng = np.random.default_rng(n)
    rows = 500
    X = rng.standard_normal((rows, n)) + 1j * rng.standard_normal((rows, n))
    O = X.conj().T @ X
    # column-major upper triangle; the lower one must not be read
    Ocm = np.ascontiguousarray(np.where(np.triu(np.ones((n, n), dtype=bool)).T, np.triu(O).T, np.nan + 0j))
    invR = np.full((n, n + 3), np.nan + 0j)
    stats = np.zeros(4)
    assert emu.emu_small_chol(_p(Ocm), ctypes.c_int64(n), n, _p(invR), ctypes.c_int64(n + 3), _p(stats)) == 0
    R = np.linalg.cholesky(O).conj().T
    got = invR[:, :n].T
    np.testing.assert_allclose(got, np.linalg.inv(R), rtol=1e-10, atol=1e-13)
    assert np.all(np.tril(got, -1) == 0)
    assert stats[0] == 1
    assert stats[1] == pytest.approx(_normest(np.linalg.inv(R)), rel=1e-10)
    assert stats[2] == pytest.approx(_normest(R), rel=1e-10)
    assert stats[3] == pytest.approx(np.linalg.norm(O), rel=1e-12)
    Xcm = np.array(X.T, order="C", copy=True)
    assert emu.emu_small_rmul(_p(Xcm), ctypes.c_int64(rows), ctypes.c_int64(rows), n, _p(np.ascontiguousarray(invR)), n + 3) == 0
    Q = Xcm.T
    np.testing.assert_allclose(Q, X @ np.linalg.inv(R), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(Q.conj().T @ Q, np.eye(n), atol=1e-12)


def test_emulated_small_cholesky_failure_modes(emu):
    """safe_cholesky (:190-210): a singular Gram matrix is shifted by alpha eps ||O|| (alpha = 100, 1000, ...) until the
    factorisation succeeds; NaN input fails all five attempts."""
    rng = np.random.default_rng(0)
    n = 6
    X = rng.standard_normal((50, n)) + 1j * rng.standard_normal((50, n))
    X[:, 3] = X[:, 1]                                        # exactly rank deficient
    O = X.conj().T @ X
    Ocm = np.ascontiguousarray(O.T)
    invR = np.zeros((n, n), dtype=complex)
    stats = np.zeros(4)
    assert emu.emu_small_chol(_p(Ocm), ctypes.c_int64(n), n, _p(invR), ctypes.c_int64(n), _p(stats)) == 0
    assert stats[0] >= 1
    nchol = int(stats[0])
    shift = sum(100.0 * 10 ** a for a in range(nchol - 1)) * np.finfo(float).eps * np.linalg.norm(O)
    Rg = np.linalg.inv(invR.T)                               # the factor that was inverted (ill-conditioned: compare R'R)
    np.testing.assert_allclose(Rg.conj().T @ Rg, O + shift * np.eye(n), atol=1e-9 * np.linalg.norm(O))
    assert stats[1] > 1e3                                     # huge growth factor: the caller loops again
    Ocm[2, 2] = np.nan
    assert emu.emu_small_chol(_p(Ocm), ctypes.c_int64(n), n, _p(invR), ctypes.c_int64(n), _p(stats)) == 0
    assert stats[0] == 0


@pytest.mark.parametrize("n", [1, 2, 7, 14, 21, 36, 45, 96])
def test_emulated_small_heev_matches_numpy(emu, n):
    """k_small_heev = the Rayleigh-Ritz eigensolver of the batched small path (eigen(Hermitian(XAX)),
    lobpcg_hyper_impl.jl:141-171): parallel cyclic Jacobi in one CTA.  Eigenvalues ascending, eigenvectors orthonormal to
    machine precision (the reference re-orthogonalises LAPACK's vectors for exactly this property), A V = V diag(w);
    only the upper triangle of the input is read; degenerate and indefinite spectra."""
    rng = np.random.default_rng(n)
    B = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))
    A = (B + B.conj().T) / 2
    if n >= 7:                                   # a degenerate cluster and a tiny eigenvalue, like a converged block
        w0 = np.sort(rng.standard_normal(n))
        w0[2] = w0[3] = w0[4]
        w0[0] = 1e-13
        Q, _ = np.linalg.qr(B)
        A = (Q * w0) @ Q.conj().T
        A = (A + A.conj().T) / 2
    ld = n + 2
    G = np.full((n, ld), np.nan + 0j)            # column-major n x n with leading dimension ld: G[j, i] = A[i, j]
    for i in range(n):
        for j in range(n):
            if i <= j:
                G[j, i] = A[i, j]                # lower triangle stays NaN: must not be read
    w = np.zeros(n)
    stats = np.zeros(4)
    assert emu.emu_small_heev(_p(G), ctypes.c_int64(ld), n, _p(w), _p(stats)) == 0
    assert stats[0] >= 1, "Jacobi did not converge"
    V = G[:, :n].T.copy()
    wref = np.linalg.eigvalsh(A)
    scale = max(1.0, np.abs(wref).max())
    np.testing.assert_allclose(w, wref, atol=4e-15 * scale * max(1, n / 8))
    assert np.all(np.diff(w) >= 0)
    assert np.abs(V.conj().T @ V - np.eye(n)).max() < 5e-16 * max(n, 32)
    assert np.abs(A @ V - V * w).max() < 1e-14 * scale * max(1, n / 8)
    assert stats[0] <= 15


# ---------------------------------------------------------------------------------------------------------------
# INT8-emulated FP64 GEMM (i8emu_core.cuh; the integer scheme behind gemm_backend 4)
# ---------------------------------------------------------------------------------------------------------------
I8_MODULI = [256, 255, 253, 251, 247, 241, 239, 233, 229, 227, 223, 217, 211, 199, 197, 193, 191, 181, 179, 173]


@pytest.mark.parametrize("n_mod,K", [(12, 1000), (16, 17116), (17, 529718), (20, 4096)])
def test_emulated_i8_crt_tables(emu, n_mod, K):
    import math
    q = (ctypes.c_int * n_mod)()
    w = (ctypes.c_double * (4 * n_mod))()
    Pl = (ctypes.c_double * 4)()
    bits = emu.emu_i8_tables(n_mod, ctypes.c_int64(K), q, w, Pl)
    p = I8_MODULI[:n_mod]
    assert all(math.gcd(a, b) == 1 for i, a in enumerate(p) for b in p[i + 1:])
    P = math.prod(p)
    assert sum(int(Pl[j]) << (40 * j) for j in range(4)) == P
    for t, pt in enumerate(p):
        W = P // pt
        assert sum(int(w[4 * t + j]) << (40 * j) for j in range(4)) == W
        assert (W * q[t]) % pt == 1
    assert K * 4 ** bits <= P // 4                                 # the exact product cannot wrap
    assert bits == 61 or P // 4 < K * 4 ** (bits + 2)              # and the budget is the largest such (cap: int64)


@pytest.mark.parametrize("n_mod", [12, 14, 16, 18])
def test_emulated_i8_zgemm_matches_exact(emu, n_mod):
    """A^H B through int8 residues / int32 accumulation / CRT against exact rational arithmetic on the same FP64 inputs;
    inputs with the dynamic range of projector tables and orbital coefficients (17 orders of magnitude)."""
    import math
    rng = np.random.default_rng(n_mod)
    k, m, n = 3000, 5, 4
    decay = np.exp(-np.linspace(0, 38, k))[:, None]
    A = (rng.standard_normal((k, m)) + 1j * rng.standard_normal((k, m))) * decay * rng.uniform(1e-3, 1e3, (1, m))
    B = (rng.standard_normal((k, n)) + 1j * rng.standard_normal((k, n))) * np.sqrt(decay) * rng.uniform(1e-2, 1e2, (1, n))
    Acm, Bcm = np.ascontiguousarray(A.T), np.ascontiguousarray(B.T)
    C = np.zeros((n, m), dtype=complex)
    bits = emu.emu_i8_zgemm_cn(n_mod, ctypes.c_int64(m), ctypes.c_int64(n), ctypes.c_int64(k), _p(Acm), _p(Bcm), _p(C))
    from fractions import Fraction
    fr = lambda x: Fraction(float(x))
    exact = np.zeros((m, n), dtype=complex)
    bound = np.zeros((m, n))
    for i in range(m):
        for j in range(n):
            re = sum(fr(A[r, i].real) * fr(B[r, j].real) + fr(A[r, i].imag) * fr(B[r, j].imag) for r in range(k))
            im = sum(fr(A[r, i].real) * fr(B[r, j].imag) - fr(A[r, i].imag) * fr(B[r, j].real) for r in range(k))
            exact[i, j] = complex(float(re), float(im))
            # truncation of both operands to `bits` bits relative to their column maxima
            bound[i, j] = 2 * k * 2.0 ** (1 - bits) * np.abs(A[:, i]).max() * np.abs(B[:, j]).max() * 2
    err = np.abs(C.T - exact)
    assert np.all(err <= bound + 1e-300), (bits, (err / bound).max())
    if n_mod >= 16:      # as accurate as an FP64 GEMM on these inputs
        ref = A.conj().T @ B
        assert err.max() <= 4 * np.abs(ref - exact).max() + 1e-18 * np.abs(exact).max()


def test_emulated_i8_update_product_matches_exact(emu):
    """C = A B (update type: the P (D P' psi) half of the nonlocal term, K = n_proj) through int8 residues with one scale
    per row of A and per column of B, against exact rational arithmetic."""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    m, k, n = 40, 130, 6
    A = (rng.standard_normal((m, k)) + 1j * rng.standard_normal((m, k))) * np.exp(-np.linspace(0, 25, m))[:, None]
    B = (rng.standard_normal((k, n)) + 1j * rng.standard_normal((k, n))) * rng.uniform(1e-4, 1e2, (1, n))
    Acm, Bcm = np.ascontiguousarray(A.T), np.ascontiguousarray(B.T)         # column-major m x k and k x n
    C = np.zeros((n, m), dtype=complex)
    bits = emu.emu_i8_zgemm_nn(16, ctypes.c_int64(m), ctypes.c_int64(n), ctypes.c_int64(k), _p(Acm), _p(Bcm), _p(C))
    assert bits >= 55
    fr = lambda x: Fraction(float(x))
    for i in range(0, m, 7):
        for j in range(n):
            re = sum(fr(A[i, r].real) * fr(B[r, j].real) - fr(A[i, r].imag) * fr(B[r, j].imag) for r in range(k))
            im = sum(fr(A[i, r].real) * fr(B[r, j].imag) + fr(A[i, r].imag) * fr(B[r, j].real) for r in range(k))
            ex = complex(float(re), float(im))
            tol = 4 * k * 2.0 ** (1 - bits) * np.abs(A[i]).max() * np.abs(B[:, j]).max()
            assert abs(C[j, i] - ex) <= tol
            assert abs(C[j, i] - ex) <= 4 * abs((A @ B)[i, j] - ex) + 1e-17 * np.abs(A[i]).max() * np.abs(B[:, j]).max() * k


def test_emulated_i8_residue_fast_equals_integer_remainder(emu):
    """a - p rint(a / p) by FMAs == symmetric 64-bit integer remainder, for integer-valued doubles up to 2^61 (53 significant
    bits), including values at +-p/2 and multiples of the moduli."""
    rng = np.random.default_rng(0)
    vals = []
    for bits in (8, 20, 40, 52, 53, 57, 61):
        mant = rng.integers(-(1 << min(bits, 53)), 1 << min(bits, 53), size=4000).astype(np.float64)
        vals.append(mant * 2.0 ** max(0, bits - 53))
    edge = []
    for p in I8_MODULI:
        for mult in (1, 2, 3, 12345, 1 << 30, (1 << 52) // p):
            base = float(p) * mult
            edge += [base, base + p // 2, base - p // 2, base + (p - 1) // 2, -base, -base - p // 2, -base + p // 2, base + 1, base - 1]
    a = np.ascontiguousarray(np.concatenate(vals + [np.array(edge)]))
    assert np.all(a == np.rint(a))
    emu.emu_i8_residue_compare.restype = ctypes.c_int64
    assert emu.emu_i8_residue_compare(ctypes.c_int64(a.size), _p(a)) == 0
