"""The LOBPCG twin (oracle/lobpcg.py) and the one-CTA Cholesky / Jacobi bodies of the small path (lobpcg_small.cuh, run
on the host through tests/hostemu/emu.cu) against the independent reference of tests/lobpcg_reference.py: a dense
diagonalisation of the same Hamiltonian, at the band-count, locking and spectrum edges.  No GPU."""
import ctypes

import numpy as np
import pytest

import lobpcg_reference as lr
from test_hostemu_fft import emu          # noqa: F401  (the host-emulation library, built by the fixture of that module)
from oracle import lobpcg as olob

EPS = np.finfo(float).eps
TOL = 1e-9
NB = (1, 2, 7, 32, 33)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module", autouse=True)
def _few_blas_threads():
    """The matrices here have a few hundred rows: a BLAS team on every core spends its time spinning (measured: 7 CPU-minutes
    for one minute of wall time on 8 cores).  Two threads for this module where threadpoolctl is installed."""
    try:
        from threadpoolctl import threadpool_limits
    except ImportError:
        yield
        return
    with threadpool_limits(limits=2):
        yield


# ---------------------------------------------------------------------------------------------------------------
# the reference checks itself
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(lr.CASES))
def test_dense_h_is_hermitian(name):
    case, H, spec = lr.problem(name, 7)
    assert H.shape == (len(case.mapping),) * 2
    assert np.abs(H - H.conj().T).max() <= 1e-14 * max(1.0, spec.norm)
    assert np.all(np.diff(case.mapping) > 0) and case.mapping[-1] < np.prod(case.fft_size)


@pytest.mark.parametrize("ik", [0, 1])
def test_dense_h_equals_oracle_block_on_identity(ik):
    case, H, spec = lr.problem(("si-gamma", "si-k")[ik], 7)
    blk = lr.silicon_oracle_block(ik)
    Ho = blk.matmul(np.eye(H.shape[0], dtype=complex))
    assert np.abs(H - Ho).max() <= 1e-12 * spec.norm


def test_exact_finds_the_multiplets():
    _, H, spec = lr.problem("diag-degenerate", 7)
    sizes = [e - s for s, e in spec.multiplets[:8]]
    assert sizes == [1, 2, 3, 6, 1, 2, 3, 6]
    _, H, spec = lr.problem("near-degenerate", 7)
    # 1e-10 splittings chain into one multiplet, 1e-6 splittings do not
    assert [e - s for s, e in spec.multiplets[:4]] == [1, 2, 3, 6]
    assert [e - s for s, e in spec.multiplets[4:16]] == [1] * 12
    _, H, spec = lr.problem("si-gamma", 7)
    # the 3-fold valence level of silicon at Gamma (degenerate up to what the 20^3 grid keeps of the symmetry)
    assert spec.w[3] - spec.w[1] < 1e-6 < min(spec.w[1] - spec.w[0], spec.w[4] - spec.w[3])
    _, H, spec = lr.problem("wide-range", 7)
    assert spec.w[0] < 0 < spec.w[-1]


def test_check_solution_rejects_wrong_answers():
    """The checker itself: the exact eigenpairs pass; a permutation of lambda without X, a rotated multiplet member
    mixed with its neighbour level, a wrong reported residual and a skipped eigenvalue are all caught."""
    nb = 7
    _, H, spec = lr.problem("diag-degenerate", nb)
    good = dict(λ=spec.w[:nb].copy(), residual_norms=np.full(nb, 1e-13), converged=True, n_iter=0, n_matvec=nb)
    X = spec.U[:, :nb].copy()
    X[:, 1:3] = X[:, 1:3] @ np.linalg.qr(np.random.default_rng(0).standard_normal((2, 2)))[0]   # inside a multiplet: fine
    good["residual_norms"] = np.linalg.norm(H @ X - X * good["λ"], axis=0) + 1e-300
    lr.check_solution(H, good, X, nb, nb, TOL, spec=spec)
    bad = dict(good, λ=good["λ"][[0, 3, 2, 1, 4, 5, 6]])
    with pytest.raises(AssertionError):
        lr.check_solution(H, bad, X, nb, nb, TOL, spec=spec)
    Xs = X[:, [3, 1, 2, 0, 4, 5, 6]]                                       # X permuted, lambda not
    with pytest.raises(AssertionError):
        lr.check_solution(H, good, Xs, nb, nb, TOL, spec=spec)
    Xm = X.copy()
    c, s = np.cos(1e-6), np.sin(1e-6)
    Xm[:, 0], Xm[:, 1] = c * X[:, 0] + s * X[:, 1], -s * X[:, 0] + c * X[:, 1]
    with pytest.raises(AssertionError):
        lr.check_solution(H, good, Xm, nb, nb, TOL, spec=spec)
    with pytest.raises(AssertionError):
        lr.check_solution(H, dict(good, residual_norms=good["residual_norms"] + 1e-8), X, nb, nb, TOL, spec=spec)
    Xk = np.concatenate([X[:, :6], spec.U[:, 12:13]], axis=1)               # eigenvalue 6 skipped for number 12
    skipped = dict(good, λ=np.concatenate([spec.w[:6], spec.w[12:13]]))
    skipped["residual_norms"] = np.linalg.norm(H @ Xk - Xk * skipped["λ"], axis=0) + 1e-300
    with pytest.raises(AssertionError):
        lr.check_solution(H, skipped, Xk, nb, nb, TOL, spec=spec)
    lr.check_solution(H, skipped, Xk, nb, nb, TOL, spec=spec, expected=[0, 1, 2, 3, 4, 5, 12])


# ---------------------------------------------------------------------------------------------------------------
# the NumPy twin against the dense diagonalisation
# ---------------------------------------------------------------------------------------------------------------
def n_conv_check_for(name, nb):
    """All bands, except at Gamma with 32 and more silicon bands: the highest ones sit in a dense part of the spectrum and
    are left as unconverged extra bands (the AdaptiveBands usage)."""
    return nb - 6 if (name == "si-gamma" and nb >= 32) else nb


# without a preconditioner these converge within 200 iterations; the other cases then exercise the maxiter return
CONVERGES_UNPRECONDITIONED = ("si-k", "tight+1", "tight+5")


def _oracle_solve(name, nb, kind, prec, maxiter=None, stats=None):
    if maxiter is None:
        # how fast the 1e-6-split clusters resolve depends on the rounding of the BLAS in use (97 to more than 200 iterations
        # for 33 bands with one and the same code)
        maxiter = 600 if name == "near-degenerate" else 200
    case, H, spec = lr.problem(name, nb)
    X0, expected, n_exact = lr.start_block(kind, spec, nb)
    ncc = n_conv_check_for(name, nb)
    miniter = 1 if kind == "random" else 0
    res = olob.lobpcg(lr.DenseOperator(H), X0.copy(), olob.PreconditionerTPA(case.kin) if prec else None, tol=TOL,
                      maxiter=maxiter, miniter=miniter, n_conv_check=ncc, stats=stats)
    return case, H, spec, res, expected, n_exact, ncc, miniter


@pytest.mark.parametrize("prec", [True, False])
@pytest.mark.parametrize("kind", lr.START_KINDS)
@pytest.mark.parametrize("nb", NB)
@pytest.mark.parametrize("name", list(lr.CASES))
def test_oracle_lobpcg_against_dense_diagonalisation(name, nb, kind, prec):
    """oracle.lobpcg.lobpcg, the twin the GPU tests compare iteration counts with, through check_solution.  A column
    locked before the last iteration reports a residual norm of exactly 0.0, as in the reference
    (lobpcg_hyper_impl.jl:367 zero-initialised history, :445 only the active rows are written, :336 the last column is
    returned); check_solution asserts that its true residual is nevertheless below tol."""
    if not prec and (kind in ("exact", "exact-high-first") or nb in (2, 32) or (name == "wide-range" and nb > 7)):
        pytest.skip("the unpreconditioned solves are paired with random and partly exact starts at 1, 7 and 33 bands")
    if nb == 2 and kind in ("exact", "partly-exact"):
        pytest.skip("two bands are run from the random start and from the one whose first column must be moved")
    if kind == "exact-high-first" and n_conv_check_for(name, nb) < nb:
        pytest.skip("`converged` is taken over the sorted columns: with unconverged extra bands the moved column pushes one of them in")
    case, H, spec, res, expected, n_exact, ncc, miniter = _oracle_solve(name, nb, kind, prec)
    X = res["X"]
    lr.check_solution(H, res, X, nb, ncc, TOL, spec=spec, expected=expected)
    if prec or name in CONVERGES_UNPRECONDITIONED or kind == "exact":
        assert res["converged"], (res["n_iter"], res["residual_norms"])
    if kind == "exact":
        assert res["n_iter"] == 0 and res["n_matvec"] == nb
        assert np.all(res["residual_norms"] < TOL)
    assert res["n_matvec"] == lr.matvecs_from_history(res["residual_history"])
    if kind == "partly-exact" and res["n_iter"] > 0:
        # the exact columns lock together at iteration 0 and report 0.0 afterwards
        assert np.all(res["residual_norms"][:n_exact] == 0.0)
        assert res["n_matvec"] <= nb + res["n_iter"] * (nb - n_exact)
    if kind == "exact-high-first" and nb > 1 and res["converged"]:
        lr.check_moved_column(H, res, X, spec, expected[-1])


# ---------------------------------------------------------------------------------------------------------------
# host emulation of the one-CTA kernels on the matrices the solver produces
# ---------------------------------------------------------------------------------------------------------------
def _record(name, nb, kind="random", prec=True):
    """Every Gram matrix handed to safe_cholesky and every Rayleigh-Ritz matrix of one oracle solve."""
    grams, rrs = [], []
    chol0, rr0 = olob.safe_cholesky, olob.rayleigh_ritz

    def chol(O, nchol=0, alpha=100.0):
        if nchol == 0:
            grams.append(np.array(O))
        return chol0(O, nchol, alpha)

    def rr(Y, AY, N):
        rrs.append(np.array(Y.conj().T @ AY))
        return rr0(Y, AY, N)
    olob.safe_cholesky, olob.rayleigh_ritz = chol, rr
    try:
        _oracle_solve(name, nb, kind, prec, maxiter=60)
    finally:
        olob.safe_cholesky, olob.rayleigh_ritz = chol0, rr0
    return grams, rrs


def _ld(x):
    return np.asarray(x, dtype=np.clongdouble)


RECORDED = [("tight+1", 7), ("tight+1", 32), ("tight+5", 2), ("near-degenerate", 32), ("near-degenerate", 7),
            ("diag-degenerate", 32), ("diag-degenerate", 1)]


@pytest.mark.parametrize("name,nb", RECORDED)
def test_emulated_cholesky_on_recorded_gram_matrices(emu, name, nb):
    """small_chol_cta on every Gram matrix of a solve (up to 32 x 32; near convergence of the tight cases their condition
    number passes 1e12 and the shifted retries happen for real).  With s the shift in use, R'R = O + s I + E and
    invR = R^-1 (I + F), ||E|| <~ n eps ||O||, ||F|| <~ n eps cond(R), so
        ||invR' O invR - I|| <= (s + 20 n eps ||O||) ||invR||^2 + 4 n eps ||R|| ||invR||.
    The attempt count is that of a NumPy replay of the five-shift rule (shift += alpha eps ||O||, alpha = 100, 1000, ...)
    wherever the replay is not decided by rounding: an attempt whose shifted matrix has its smallest eigenvalue within
    20 n eps ||O|| of zero may go either way."""
    grams, _ = _record(name, nb)
    assert grams
    worst_cond, retried = 1.0, 0
    for O in grams:
        n = O.shape[0]
        Oh = np.triu(O) + np.triu(O, 1).conj().T
        onorm = np.linalg.norm(Oh)
        Ocm = np.ascontiguousarray(np.where(np.triu(np.ones((n, n), dtype=bool)).T, np.triu(Oh).T, np.nan + 0j))
        invR = np.full((n, n), np.nan + 0j)
        stats = np.zeros(4)
        assert emu.emu_small_chol(_p(Ocm), ctypes.c_int64(n), n, _p(invR), ctypes.c_int64(n), _p(stats)) == 0
        nchol = int(stats[0])
        assert 1 <= nchol <= 5
        assert stats[3] == pytest.approx(onorm, rel=1e-13)
        # replay of the shift rule
        lam_min = np.linalg.eigvalsh(Oh)[0]
        margin = 20 * n * EPS * onorm
        shifts = np.concatenate([[0.0], np.cumsum([100.0 * 10 ** a * EPS * onorm for a in range(4)])])
        lo = next((k + 1 for k in range(5) if lam_min + shifts[k] > -margin), 6)    # earliest attempt that may succeed
        hi = next((k + 1 for k in range(5) if lam_min + shifts[k] > margin), 6)     # attempt that must succeed
        assert lo <= nchol <= hi, (nchol, lo, hi, lam_min / onorm)
        retried += nchol > 1
        s = shifts[nchol - 1]
        Ri = invR.T                                      # column-major n x n -> invR
        assert np.all(np.tril(Ri, -1) == 0)
        ninv = np.linalg.norm(Ri, 2)
        res = np.asarray(_ld(Ri).conj().T @ _ld(Oh) @ _ld(Ri) - np.eye(n), dtype=complex)
        nR = np.linalg.norm(np.linalg.inv(Ri), 2)
        bound = (s + 20 * n * EPS * onorm) * ninv ** 2 + 4 * n * EPS * nR * ninv
        assert np.linalg.norm(res, 2) <= bound, (np.linalg.norm(res, 2), bound, nchol)
        worst_cond = max(worst_cond, np.linalg.cond(Oh))
        assert stats[1] == pytest.approx(olob.normest(Ri), rel=1e-9)
        # X invR through small_rmul_row on a tall block with this Gram matrix
        if n <= 32 and nchol == 1 and np.linalg.cond(Oh) < 1e6:
            L = np.linalg.cholesky(Oh)
            Q = np.linalg.qr(np.random.default_rng(n).standard_normal((3 * n + 5, n)) + 0j)[0]
            Xt = Q @ L.conj().T                                        # Xt' Xt = O
            Xcm = np.array(Xt.T, order="C", copy=True)
            rows = Xt.shape[0]
            assert emu.emu_small_rmul(_p(Xcm), ctypes.c_int64(rows), ctypes.c_int64(rows), n, _p(np.ascontiguousarray(invR)), n) == 0
            got = Xcm.T
            assert np.abs(got.conj().T @ got - np.eye(n)).max() <= 50 * n * EPS * np.linalg.cond(Oh)
    if name.startswith("tight") and nb >= 7:
        assert worst_cond > 1e12 or retried, "the tight case no longer produces an ill-conditioned Gram matrix"


def _heev(emu, A):
    n = A.shape[0]
    ld = n + 1
    G = np.full((n, ld), np.nan + 0j)
    iu = np.triu_indices(n)
    G[iu[1], iu[0]] = A[iu]                             # column-major upper triangle; the lower one stays NaN
    w, stats = np.zeros(n), np.zeros(4)
    assert emu.emu_small_heev(_p(G), ctypes.c_int64(ld), n, _p(w), _p(stats)) == 0
    return w, G[:, :n].T.copy(), stats


def _check_heev(A, w, V, stats):
    n = A.shape[0]
    Ah = np.triu(A) + np.triu(A, 1).conj().T
    Ah[np.diag_indices(n)] = Ah[np.diag_indices(n)].real
    nA = np.linalg.norm(Ah)
    assert stats[0] != 0, "Jacobi did not converge within 60 sweeps"
    assert np.all(np.diff(w) >= 0)
    bound = 50 * n * EPS
    r = np.asarray(_ld(Ah) @ _ld(V) - _ld(V) * _ld(w)[None, :], dtype=complex)
    assert np.linalg.norm(r) <= bound * nA + 1e-300, (np.linalg.norm(r) / max(nA, 1e-300), bound)
    o = np.asarray(_ld(V).conj().T @ _ld(V) - np.eye(n), dtype=complex)
    assert np.linalg.norm(o) <= bound, (np.linalg.norm(o), bound)
    # Weyl: the off-diagonal remnant the sweeps stop at (2 sqrt(n) eps ||G||) moves an eigenvalue by at most its norm; LAPACK's
    # own values carry n eps ||G||
    assert np.abs(w - np.linalg.eigvalsh(Ah)).max() <= (n + 2 * np.sqrt(n) + 2) * EPS * nA


@pytest.mark.parametrize("name,nb", RECORDED)
def test_emulated_jacobi_on_recorded_rayleigh_ritz_matrices(emu, name, nb):
    """small_heev_cta on the Rayleigh-Ritz matrix of every iteration of a solve (2 nb and 3 nb columns, up to 96): near
    convergence these carry the exactly degenerate and 1e-10-split clusters of the Hamiltonian next to entries of the
    size of the residuals."""
    _, rrs = _record(name, nb)
    assert rrs and max(A.shape[0] for A in rrs) == (2 * nb if len(rrs) == 1 else 3 * nb)
    for A in rrs:
        w, V, stats = _heev(emu, A)
        _check_heev(A, w, V, stats)


@pytest.mark.parametrize("n", [1, 2, 5, 32, 33, 96])
def test_emulated_jacobi_ties_and_zero(emu, n):
    rng = np.random.default_rng(n)
    Z = np.zeros((n, n), dtype=complex)
    w, V, stats = _heev(emu, Z)
    assert stats[0] != 0 and np.all(w == 0) and np.array_equal(V, np.eye(n))
    w, V, stats = _heev(emu, 2.5 * np.eye(n) + 0j)                         # one n-fold tie
    assert stats[0] != 0 and np.all(w == 2.5) and np.array_equal(V, np.eye(n))
    if n >= 5:
        Q = np.linalg.qr(rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n)))[0]
        for split in (0.0, 1e-10):
            d = np.sort(rng.standard_normal(n))
            d[1:4] = d[1] + split * np.arange(3)
            d[-2:] = d[-1]
            d = np.sort(d)
            A = (Q * d) @ Q.conj().T
            w, V, stats = _heev(emu, A)
            _check_heev(A, w, V, stats)
            assert np.abs(w - d).max() <= 4 * n * EPS * np.abs(d).max()
