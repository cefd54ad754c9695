"""Independent reference for the LOBPCG eigensolvers (plain NumPy: no oracle, no GPU).

The device solvers (lobpcg.cu, lobpcg_small.cuh, lobpcg_batch.cuh) and their NumPy twin (oracle/lobpcg.py) state the
same algorithm, so agreement between them does not say that an eigenpair is right.  This module assembles the
Hamiltonian of a k-block as a dense matrix from the arrays the block is created from, diagonalises it with
numpy.linalg.eigh, and checks a solver result against that from first principles (`check_solution`).

Conventions (those of the C ABI, include/dftk_b200.h):
  mapping  0-based linear cube index of each plane wave, x fastest: index = x + nx (y + ny z)
  local    FFT[V . IFFT[psi]] with a normalised transform pair (dftk_b200_apply_h), i.e. S' F diag(V) F^-1 S with
           F = numpy.fft.fftn, F^-1 = numpy.fft.ifftn on the (nz, ny, nx) cube and S the zero-padding of the sphere
  P, D     n_pw x n_proj complex and n_proj x n_proj real symmetric: the nonlocal term is P D P'
Orbital blocks are n_pw x n_bands arrays (a column per band) throughout.
"""
import functools
from typing import NamedTuple, Optional

import numpy as np

EPS = np.finfo(float).eps
MULTIPLET_TOL = 1e-9


# ---------------------------------------------------------------------------------------------------------------
# dense operator
# ---------------------------------------------------------------------------------------------------------------
def dense_h(fft_size, mapping, kin, V, P, D):
    """H = diag(kin) + S' F diag(V) F^-1 S + P D P' as an n_pw x n_pw complex128 matrix.  The local term is built by
    sending identity columns through numpy.fft; any of kin, V, (P, D) may be None."""
    nx, ny, nz = (int(n) for n in fft_size)
    N = nx * ny * nz
    mapping = np.asarray(mapping, dtype=np.int64)
    n = len(mapping)
    H = np.zeros((n, n), dtype=np.complex128)
    if V is not None:
        Vc = np.asarray(V, dtype=np.float64).reshape(nz, ny, nx)
        chunk = 128
        for j0 in range(0, n, chunk):
            j1 = min(n, j0 + chunk)
            cube = np.zeros((j1 - j0, N), dtype=np.complex128)
            cube[np.arange(j1 - j0), mapping[j0:j1]] = 1.0
            real = np.fft.ifftn(cube.reshape(-1, nz, ny, nx), axes=(1, 2, 3))
            back = np.fft.fftn(real * Vc[None], axes=(1, 2, 3)).reshape(-1, N)
            H[:, j0:j1] = back[:, mapping].T
    if kin is not None:
        H[np.arange(n), np.arange(n)] += np.asarray(kin, dtype=np.float64)
    if P is not None:
        H += P @ (np.asarray(D, dtype=np.float64) @ P.conj().T)
    return H


class Spectrum(NamedTuple):
    w: np.ndarray           # all eigenvalues, ascending
    U: np.ndarray           # eigenvectors (columns)
    multiplets: list        # [(start, stop)] over the whole spectrum: runs of eigenvalues closer than MULTIPLET_TOL
    norm: float             # ||H||_2


def exact(H, nb=None):
    """numpy.linalg.eigh of H and its multiplets (chains of neighbouring eigenvalues closer than 1e-9).  With `nb` the
    values and vectors are cut to the lowest nb and the multiplets to those that start below nb."""
    Hh = (H + H.conj().T) / 2
    w, U = np.linalg.eigh(Hh)
    starts = [0] + [i for i in range(1, len(w)) if w[i] - w[i - 1] >= MULTIPLET_TOL]
    mult = [(s, e) for s, e in zip(starts, starts[1:] + [len(w)])]
    norm = float(max(abs(w[0]), abs(w[-1])))
    if nb is not None:
        return Spectrum(w[:nb], U[:, :nb], [m for m in mult if m[0] < nb], norm)
    return Spectrum(w, U, mult, norm)


class DenseOperator:
    """The dense H behind the `matmul` interface of oracle.lobpcg.lobpcg."""

    def __init__(self, H):
        self.H = H

    def matmul(self, X):
        return self.H @ X

    __matmul__ = matmul


# ---------------------------------------------------------------------------------------------------------------
# case table
# ---------------------------------------------------------------------------------------------------------------
class Case(NamedTuple):
    fft_size: tuple
    mapping: np.ndarray
    kin: Optional[np.ndarray]
    V: Optional[np.ndarray]
    P: Optional[np.ndarray]
    D: Optional[np.ndarray]
    description: str


def sphere_mapping(fft_size, n_pw):
    """The n_pw cube points of smallest |G|^2 (ties by cube index), ascending: a sphere-shaped set of any size."""
    nx, ny, nz = fft_size
    gx, gy, gz = (np.fft.fftfreq(n, 1.0 / n) for n in (nx, ny, nz))
    g2 = (gz[:, None, None] ** 2 + gy[None, :, None] ** 2 + gx[None, None, :] ** 2).reshape(-1)
    assert n_pw <= len(g2)
    return np.sort(np.argsort(g2, kind="stable")[:n_pw]).astype(np.int64)


def _random_projectors(rng, n_pw, n_proj, scale, sign):
    """Random complex P without +-q symmetry (the device stays on the complex projector products) and a block-diagonal
    real symmetric D of 3x3 blocks whose eigenvalues have the sign `sign`."""
    P = (rng.standard_normal((n_pw, n_proj)) + 1j * rng.standard_normal((n_pw, n_proj))) / np.sqrt(2 * n_pw)
    D = np.zeros((n_proj, n_proj))
    for b0 in range(0, n_proj, 3):
        m = min(3, n_proj - b0)
        A = rng.standard_normal((m, m))
        D[b0:b0 + m, b0:b0 + m] = sign * scale * (A @ A.T / m + 0.2 * np.eye(m))
    return P, D


MULTIPLET_SIZES = (1, 2, 3, 6)


def _multiplet_levels(n_levels, split):
    """Levels 1.0, 1.25, ... in multiplets of sizes 1, 2, 3, 6, 1, 2, ...: the multiplets end after 1, 3, 6, 12, 13, 15, 18,
    24, 25, 27, 30, 36, 37, 39, 42, 48, ... states, so 1, 3 and 36 bands end at an edge and 2, 7, 8, 31, 32, 33, 40 and 64
    inside one.  `split(group, j)` is added to member j of multiplet number `group`."""
    out, g = [], 0
    while len(out) < n_levels:
        for j in range(MULTIPLET_SIZES[g % 4]):
            out.append(1.0 + 0.25 * g + split(g, j))
        g += 1
    return np.array(out[:n_levels])


def _diagonal_case(nb, seed, split, what):
    rng = np.random.default_rng(seed)
    fft_size, n_pw = (12, 12, 12), 420
    n_lev = 96
    lev = _multiplet_levels(n_lev, split)
    rest = lev.max() + 0.5 + np.cumsum(0.05 + 0.1 * rng.random(n_pw - n_lev))
    kin = np.concatenate([lev, rest])[rng.permutation(n_pw)]       # multiplet members are scattered over the sphere
    V = np.zeros(int(np.prod(fft_size)))
    return Case(fft_size, sphere_mapping(fft_size, n_pw), kin, V, None, None, what)


def case_diag_degenerate(nb, seed=0):
    return _diagonal_case(nb, seed, lambda g, j: 0.0,
                          "diagonal H (V = 0, no projectors) with exact multiplets of sizes 1, 2, 3, 6")


def case_near_degenerate(nb, seed=0):
    return _diagonal_case(nb, seed, lambda g, j: j * (1e-10 if (g // 4) % 2 == 0 else 1e-6),
                          "diagonal H with multiplets split by 1e-10 and 1e-6")


def case_wide_range(nb, seed=0):
    rng = np.random.default_rng(seed + 1)
    fft_size, n_pw = (16, 16, 16), 480
    kin = np.logspace(-3, 4, n_pw)
    V = -(0.5 + 2.5 * rng.random(int(np.prod(fft_size))))
    P, D = _random_projectors(rng, n_pw, 12, 2.0, -1.0)
    return Case(fft_size, sphere_mapping(fft_size, n_pw), kin, V, P, D,
                "kin from 1e-3 to 1e4, negative V and negative D: negative eigenvalues, a hard case for TPA")


def _tight(extra):
    def make(nb, seed=0):
        rng = np.random.default_rng(seed + 2)
        fft_size, n_pw = (12, 12, 12), 3 * nb + extra
        kin = 0.5 + np.sort(4.0 * rng.random(n_pw))
        V = 0.5 * rng.standard_normal(int(np.prod(fft_size)))
        P, D = _random_projectors(rng, n_pw, 2, 1.0, 1.0)
        return Case(fft_size, sphere_mapping(fft_size, n_pw), kin, V, P, D,
                    f"n_pw = 3 nb + {extra}: the [X R P] subspace is almost the whole space")
    return make


def _many_projectors(n_proj):
    def make(nb, seed=0):
        rng = np.random.default_rng(seed + 3)
        fft_size, n_pw = (12, 12, 12), 400
        mapping = sphere_mapping(fft_size, n_pw)
        kin = 0.5 * (0.3 * np.arange(n_pw) ** (2.0 / 3.0) + 0.05 * rng.random(n_pw))
        V = 0.3 * rng.standard_normal(int(np.prod(fft_size)))
        P, D = _random_projectors(rng, n_pw, n_proj, 1.5, 1.0)
        return Case(fft_size, mapping, kin, V, P, D, f"{n_proj} projectors (96 = SMALL_MAX_COLS of the batched apply)")
    return make


@functools.lru_cache(maxsize=None)
def _silicon_blocks():
    from gpu_common import silicon_setup      # oracle-side basis data only; the dense H is assembled by dense_h
    _, b, _, _, ham = silicon_setup(Ecut=12, fft_size=(20, 20, 20), kcoords=((0.0, 0.0, 0.0), (0.1, -0.2, 0.3)),
                                    kweights=(0.5, 0.5))
    return b, ham


def _silicon(ik, what):
    def make(nb, seed=0):
        b, ham = _silicon_blocks()
        blk = ham[ik]
        return Case(tuple(b.fft_size), blk.kpt.mapping.copy(), blk.kin.copy(), np.array(blk.Vtot, dtype=float).reshape(-1),
                    np.array(blk.PD[0]), np.array(blk.PD[1]), what)
    return make


@functools.lru_cache(maxsize=None)
def large_silicon_problem():
    """(case, H, Spectrum) of a silicon block with more than 2048 plane waves (Ecut 30 on a 24^3 grid, generic k): long
    enough for the INT8 tensor-core products of gemm_backend 4 at i8_min_rows = 2048.  Not part of CASES."""
    from gpu_common import silicon_setup
    _, b, _, _, ham = silicon_setup(Ecut=30, fft_size=(24, 24, 24), kcoords=((0.1, -0.2, 0.3),), kweights=(1.0,))
    blk = ham[0]
    case = Case(tuple(b.fft_size), blk.kpt.mapping.copy(), blk.kin.copy(), np.array(blk.Vtot, dtype=float).reshape(-1),
                np.array(blk.PD[0]), np.array(blk.PD[1]), "silicon LDA block, Ecut 30, k = (0.1, -0.2, 0.3)")
    H = dense_h(*case[:6])
    return case, H, exact(H)


def silicon_oracle_block(ik):
    """The oracle's Hamiltonian block behind the `si` cases (for the self-check of dense_h)."""
    return _silicon_blocks()[1][ik]


CASES = {
    "si-gamma": _silicon(0, "silicon LDA block at Gamma (time-reversal fold of the projector products, 3-fold degeneracies)"),
    "si-k": _silicon(1, "silicon LDA block at k = (0.1, -0.2, 0.3)"),
    "diag-degenerate": case_diag_degenerate,
    "near-degenerate": case_near_degenerate,
    "wide-range": case_wide_range,
    "tight+1": _tight(1),
    "tight+5": _tight(5),
    "many-projectors-96": _many_projectors(96),
    "many-projectors-97": _many_projectors(97),
}
# cases on which the iteration count of two implementations can be compared (no rank-deficient subspaces, no clusters
# whose resolution depends on rounding)
WELL_CONDITIONED = ("si-gamma", "si-k", "diag-degenerate", "many-projectors-96", "many-projectors-97")


@functools.lru_cache(maxsize=64)
def problem(name, nb, seed=0):
    """(case, dense H, Spectrum of the whole H) of CASES[name](nb, seed), cached."""
    case = CASES[name](nb, seed)
    H = dense_h(*case[:6])
    return case, H, exact(H)


# ---------------------------------------------------------------------------------------------------------------
# start blocks
# ---------------------------------------------------------------------------------------------------------------
START_KINDS = ("random", "exact", "exact-high-first", "partly-exact")


def start_block(kind, spec, nb, seed=0):
    """(X0, expected, n_exact): the n_pw x nb start block, the indices of the exact eigenvalues the solve must return
    (ascending) and the number of leading columns that are exact eigenvectors.

    random            complex normal
    exact             the nb lowest eigenvectors: converges at iteration 0
    exact-high-first  column 0 is the exact eigenvector number nb + 3 (or the highest there is), the rest random: with
                      miniter = 0 it locks at iteration 0 and stays first while the other columns converge below it,
                      so the final sort has to move it, with its vector, to the end
    partly-exact      the first max(1, nb // 2) columns are exact: locking advances by several columns at once
    """
    n = spec.U.shape[0]
    rng = np.random.default_rng(1000 + seed)
    X0 = rng.standard_normal((n, nb)) + 1j * rng.standard_normal((n, nb))
    expected = np.arange(nb)
    n_exact = 0
    if kind == "exact":
        X0 = spec.U[:, :nb].copy()
        n_exact = nb
    elif kind == "exact-high-first":
        hi = min(nb + 3, n - 1)
        X0[:, 0] = spec.U[:, hi]
        expected = np.concatenate([np.arange(nb - 1), [hi]])
        n_exact = 1
    elif kind == "partly-exact":
        n_exact = max(1, nb // 2)
        X0[:, :n_exact] = spec.U[:, :n_exact]
    elif kind != "random":
        raise ValueError(kind)
    return X0, expected, n_exact


# ---------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------
def matvecs_from_history(hist):
    """Number of H applications implied by a residual history (nb x (n_iter + 1), rows in any order): nb for the start
    block, then one per column still active at each iteration (lobpcg_hyper_impl.jl:416).  The history holds a norm for
    the active columns of an iteration and exactly 0.0 for the locked ones (:367,445)."""
    return hist.shape[0] + int(np.count_nonzero(hist[:, 1:]))


def _multiplet_of(spec, i):
    for s, e in spec.multiplets:
        if s <= i < e:
            return s, e
    raise IndexError(i)


def check_solution(H, res, X, nb, n_conv_check, tol, *, spec=None, expected=None, drift=None):
    """Assert from first principles that `res` (the dict of KBlock.lobpcg / oracle.lobpcg.lobpcg) with the n_pw x nb
    block X is a solution of the eigenproblem of the dense Hermitian H.  Returns the true residual norms.

    * X'X = I to max(1e-12, 3 nb (n_iter + 1) eps), lambda ascending, lambda_c = Rayleigh quotient of column c to 1e-11 ||H||.
    * `converged` is what the reported norms say: max residual_norms[:n_conv_check] < tol.
    * If converged, the true residual ||H x_c - lambda_c x_c|| of every c < n_conv_check is below tol + drift.  The
      solvers never re-apply H to X: H X is carried through the products (AY) cX, each of which adds a rounding error
      of the order 3 nb eps ||H||, so the carried residual and the true one drift apart by that per iteration:
      drift = 3 nb (n_iter + 1) eps ||H|| (3e-12 for 8 silicon bands after 50 iterations).
    * Every lambda_c, converged or not, lies within the true residual of an exact eigenvalue (the residual bound of a
      Rayleigh quotient).  If converged, lambda_c is within it of eigenvalue number expected[c] (default c: no
      eigenvalue is skipped), and within ||r||^2 / gap of it (Kato-Temple), gap being the distance of lambda_c to the
      exact spectrum outside the multiplet of that eigenvalue; the width of the multiplet is added to both.
    * For every multiplet wholly inside the converged columns, the returned columns span the exact eigenspace:
      ||sin Theta|| <= 10 ||R||_F / gap (Davis-Kahan), a subspace check and never a per-vector one.
    * residual_norms[c] equals the true residual to 1e-6 of it plus drift for the columns active at the last iteration
      (a column that reports 0.0 is taken as locked earlier; that the locked columns do report 0.0 is asserted by the
      tests that know which columns lock, not here).  A column
      locked at an earlier iteration reports exactly 0.0: the residual history starts as zeros, an iteration writes
      the rows of its active columns only, and the result is the column of the last iteration
      (lobpcg_hyper_impl.jl:367,445,336).  Such a column was locked under tol and is not touched again, so its true
      residual must still be below tol + drift.
    """
    spec = exact(H) if spec is None else spec
    w, U = spec.w, spec.U
    normH = spec.norm
    n = H.shape[0]
    if drift is None:
        drift = 3 * nb * (int(res["n_iter"]) + 1) * EPS * max(normH, 1.0)
    slack = 1e-12 * max(normH, 1.0)            # accuracy of the dense diagonalisation itself
    expected = np.arange(nb) if expected is None else np.asarray(expected)
    lam = np.asarray(res["λ"], dtype=float)
    rn = np.asarray(res["residual_norms"], dtype=float)
    assert X.shape == (n, nb) and lam.shape == (nb,) and rn.shape == (nb,)
    assert np.all(np.isfinite(X)) and np.all(np.isfinite(lam)) and np.all(np.isfinite(rn))

    G = X.conj().T @ X
    # X is never re-orthonormalised against itself: each X <- Y cX carries the rounding of a product with up to 3 nb
    # columns, so the defect may grow by 3 nb eps per iteration (1e-12 covers every solve but the longest many-band ones)
    orth_tol = max(1e-12, 3 * nb * (int(res["n_iter"]) + 1) * EPS)
    assert np.abs(G - np.eye(nb)).max() <= orth_tol, f"X'X - I = {np.abs(G - np.eye(nb)).max():.3e} > {orth_tol:.3e}"
    assert np.all(np.diff(lam) >= 0), f"eigenvalues not ascending: {lam}"
    HX = H @ X
    rq = np.real(np.sum(X.conj() * HX, axis=0)) / np.real(np.sum(X.conj() * X, axis=0))
    assert np.abs(lam - rq).max() <= 1e-11 * max(normH, 1.0), \
        f"lambda is not the Rayleigh quotient of its column: {np.abs(lam - rq).max():.3e} (||H|| = {normH:.3e})"
    true_r = np.linalg.norm(HX - X * lam[None, :], axis=0)

    converged = bool(res["converged"])
    assert converged == bool(rn[:n_conv_check].max() < tol), (converged, rn[:n_conv_check].max(), tol)

    # reported residual norms
    for c in range(nb):
        if rn[c] == 0.0:
            assert true_r[c] < tol + drift, f"column {c} reports 0.0 (locked earlier) but its true residual is {true_r[c]:.3e}"
        else:
            assert abs(rn[c] - true_r[c]) <= 1e-6 * true_r[c] + drift, \
                f"column {c}: reported residual {rn[c]:.3e}, true {true_r[c]:.3e} (drift allowance {drift:.3e})"

    # eigenvalues
    nearest = np.abs(lam[:, None] - w[None, :]).min(axis=1)
    assert np.all(nearest <= true_r + slack), f"lambda farther from the spectrum than its residual: {nearest} vs {true_r}"
    if converged:
        ncc = n_conv_check
        assert np.all(true_r[:ncc] < tol + drift), f"true residuals {true_r[:ncc]} exceed tol = {tol}"
        for c in range(ncc):
            s, e = _multiplet_of(spec, int(expected[c]))
            width = w[e - 1] - w[s]
            err = abs(lam[c] - w[expected[c]])
            assert err <= true_r[c] + width + slack, \
                f"column {c}: lambda = {lam[c]!r}, eigenvalue {expected[c]} = {w[expected[c]]!r}, residual {true_r[c]:.3e}"
            outside = np.concatenate([w[:s], w[e:]])
            if len(outside):
                gap = np.abs(outside - lam[c]).min()
                if gap > 2 * true_r[c]:
                    assert err <= true_r[c] ** 2 / gap + width + slack, \
                        f"column {c}: |lambda - exact| = {err:.3e} > r^2/gap = {true_r[c] ** 2 / gap:.3e}"
        # eigenspaces of the multiplets wholly inside the converged columns
        for s, e in spec.multiplets:
            if e > ncc:
                break
            if not np.array_equal(expected[s:e], np.arange(s, e)):
                continue
            gap = min(w[s] - w[s - 1] if s > 0 else np.inf, w[e] - w[e - 1] if e < n else np.inf)
            Xm, Um = X[:, s:e], U[:, s:e]
            sin_theta = np.linalg.norm(Xm - Um @ (Um.conj().T @ Xm), 2)
            Rm = np.linalg.norm(true_r[s:e])
            bound = 10 * (Rm + slack) / gap + 1e-12
            assert sin_theta <= bound, f"multiplet {s}:{e}: sin(theta) = {sin_theta:.3e} > {bound:.3e} (gap {gap:.3e})"
    if res["n_iter"] == 0:
        assert res["n_matvec"] == nb
    else:
        assert nb + res["n_iter"] <= res["n_matvec"] <= nb * (1 + res["n_iter"])
    return true_r


def check_moved_column(H, res, X, spec, hi):
    """After an `exact-high-first` solve: the start column that was the exact eigenvector number `hi` locked first (at
    iteration 0, with miniter = 0) and was never touched again, so it is still in X, to rounding, at the sorted position
    of its eigenvalue -- among the last columns (other columns may have converged into the same multiplet) -- with
    lambda = w[hi], and it reports 0.0 when the solve went on after iteration 0.  A sort that moves lambda but not X
    leaves it in column 0."""
    lam = np.asarray(res["λ"])
    overlap = np.abs(spec.U[:, hi].conj() @ X)
    j = int(np.argmax(overlap))
    assert overlap[j] >= 1 - 1e-12, f"the locked eigenvector is no longer a column of X (best overlap {overlap[j]!r})"
    assert abs(lam[j] - spec.w[hi]) <= 1e-11 * max(1.0, spec.norm), (j, lam[j], spec.w[hi])
    s, e = _multiplet_of(spec, hi)
    assert j >= len(lam) - (e - s), f"column {j} of {len(lam)} holds the highest eigenvalue"
    if res["n_iter"] > 0:
        assert res["residual_norms"][j] == 0.0
