"""Plain reference of the pruned sphere<->cube transforms (NumPy only, no GPU): an ellipsoid sphere generator and a direct
separable DFT that does not share any factorisation with the FFT engines under test.

Conventions (those of oracle/basis.py ifft_kpt / fft_kpt and of the device calls):
  cubes are flat, x fastest (shape (nz, ny, nx) when reshaped); F is the unnormalised forward DFT (sign -1) and
  F^-1 = (1/N) * (unnormalised backward DFT), so N F^-1 is the unnormalised backward transform.
  - local apply:    gather(F diag(V) F^-1 scatter psi) + kin psi
  - sphere_to_real: ifft_norm N F^-1 scatter psi
  - real_to_sphere: fft_norm gather(F f)
  - density:        sum_n w_n ifft_norm^2 |N F^-1 scatter psi_n|^2
"""
import os
import re

import numpy as np

FFT_PLAN_H = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "dftk.jl_b200", "csrc", "fft_plan.h")

# an off-centre k-point: the sphere is asymmetric and wraps, so every axis has two index ranges
K_OFF = (0.3, -0.2, 0.45)
# frac of a sphere that fills the whole box: sqrt(3) (1/2 + max|k|/n) / (1/2) < 2 for every axis length >= 8
FULL = 2.0
HALF = 0.5
_PI = np.longdouble("3.141592653589793238462643383279502884197")


def centred_freqs(n):
    """Integer frequencies of the n points of an axis in FFT order: 0, 1, ..., -2, -1 (DFTK's G_vectors)."""
    j = np.arange(n)
    return np.where(j <= (n - 1) // 2, j, j - n)


def ellipsoid_mapping(shape_xyz, frac, k=K_OFF):
    """0-based linear cube indices (x fastest, ascending) of the points with sum_i ((g_i + k_i) / (frac n_i / 2))^2 <= 1.
    frac = 0 gives the one-point sphere {G = 0}."""
    if frac == 0:
        return np.zeros(1, dtype=np.int64)
    nx, ny, nz = shape_xyz
    gz, gy, gx = np.meshgrid(*[centred_freqs(n) for n in (nz, ny, nx)], indexing="ij")
    r2 = sum(((g + ki) / (frac * n / 2.0)) ** 2 for g, ki, n in ((gx, k[0], nx), (gy, k[1], ny), (gz, k[2], nz)))
    return np.flatnonzero(r2.reshape(-1) <= 1.0).astype(np.int64)


def dft_matrix(n, sign):
    """M[j, m] = exp(sign 2 pi i j m / n), phases reduced exactly in integers, cos / sin in long double."""
    j = np.arange(n, dtype=np.int64)
    ph = np.outer(j, j) % n
    ang = (2 * _PI / n) * ph.astype(np.longdouble)
    return (np.cos(ang).astype(np.float64) + sign * 1j * np.sin(ang).astype(np.float64))


def dft3(data, shape_xyz, sign):
    """Unnormalised 3D DFT with exponent sign `sign` of flat cubes data[..., N] (x fastest), one axis at a time."""
    nx, ny, nz = shape_xyz
    lead = data.shape[:-1]
    c = np.asarray(data, dtype=np.complex128).reshape(lead + (nz, ny, nx))
    for ax, n in ((-1, nx), (-2, ny), (-3, nz)):
        t = np.ascontiguousarray(np.moveaxis(c, ax, -1))
        t = (t.reshape(-1, n) @ dft_matrix(n, sign)).reshape(t.shape)                # the matrix is symmetric
        c = np.moveaxis(t, -1, ax)
    return np.ascontiguousarray(c).reshape(lead + (nx * ny * nz,))


def scatter(psi, mapping, shape_xyz):
    """Zero-padded cubes of sphere coefficients psi[..., n_pw]."""
    out = np.zeros(psi.shape[:-1] + (int(np.prod(shape_xyz)),), dtype=np.complex128)
    out[..., mapping] = psi
    return out


def local_apply(psi, mapping, shape_xyz, V, kin=None):
    """gather(F diag(V) F^-1 scatter psi) (+ kin psi)."""
    N = int(np.prod(shape_xyz))
    real = dft3(scatter(psi, mapping, shape_xyz), shape_xyz, +1) / N
    out = dft3(real * V, shape_xyz, -1)[..., mapping]
    return out if kin is None else out + kin * psi


def sphere_to_real(psi, mapping, shape_xyz, ifft_norm=1.0):
    return ifft_norm * dft3(scatter(psi, mapping, shape_xyz), shape_xyz, +1)


def real_to_sphere(f, mapping, shape_xyz, fft_norm=1.0):
    return fft_norm * dft3(f, shape_xyz, -1)[..., mapping]


def density(psi, weights, mapping, shape_xyz, ifft_norm=1.0):
    cube = sphere_to_real(psi, mapping, shape_xyz, ifft_norm)
    return np.einsum("n,nr->r", np.asarray(weights, dtype=np.float64), np.abs(cube) ** 2)


def reg_pairs():
    """The factor pairs (A, B) of the register two-pass engine, read from DFTK_REG_PAIRS in fft_plan.h."""
    with open(FFT_PLAN_H) as f:
        src = f.read()
    body = re.search(r"#define DFTK_REG_PAIRS\(X\)((?:[^\n]*\\\n)*[^\n]*)", src).group(1)
    pairs = [(int(a), int(b)) for a, b in re.findall(r"X\((\d+),\s*(\d+)\)", body)]
    assert pairs and len({a * b for a, b in pairs}) == len(pairs), pairs
    return pairs


def placements(n):
    """An axis length n on x, y and z of a box whose other extents (18, 25) are not multiples of the engines' line
    counts, so the x tiles of the y / z stages are ragged."""
    return {"x": (n, 18, 25), "y": (25, n, 18), "z": (18, 25, n)}


def index_runs(present):
    """Number of maximal runs of True in a 1D boolean array (no wrap-around)."""
    p = np.asarray(present, dtype=np.int8)
    return int(np.sum(np.diff(np.concatenate([[0], p])) == 1))
