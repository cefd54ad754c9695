"""Independent NumPy restatement of the basis transfers (test infrastructure only; the package never imports it):
transfer_mapping (transfer.jl:10-83), apply_symop (symmetry.jl:229-270), the Fourier block copy of transfer_density
(transfer.jl:165-178), cell_to_supercell(ψ, ...) (supercell.jl:58-93) and the periodic quadratic B-spline of
interpolate_density (Interpolations.jl BSpline(Quadratic(Periodic(OnCell())))).

Written from the Julia formulas with 1-based ranges converted once; orbitals are (n_G, n_bands) as in the oracle, cubes are
arrays indexed [z, y, x] (x fastest in the flat order)."""
import math

import numpy as np

from oracle.basis import index_G_vectors, normalize_kpoint_coordinate


def transfer_mapping_grid(fft_in, fft_out):
    """The 8 (block_in, block_out) pairs of per-axis (x, y, z) 0-based ranges."""
    per_axis = []
    for n_in, n_out in zip(fft_in, fft_out):
        if n_in <= n_out:
            a, b = math.ceil(n_in / 2), n_in // 2
            per_axis.append(((range(0, a), range(a, n_in)), (range(0, a), range(n_out - b, n_out))))
        else:
            a, b = math.ceil(n_out / 2), n_out // 2
            per_axis.append(((range(0, a), range(n_in - b, n_in)), (range(0, a), range(a, n_out))))
    pairs = []
    for i in range(2):
        for j in range(2):
            for k in range(2):
                pairs.append(((per_axis[0][0][i], per_axis[1][0][j], per_axis[2][0][k]),
                              (per_axis[0][1][i], per_axis[1][1][j], per_axis[2][1][k])))
    return pairs


def block_copy(f_in, fft_in, fft_out):
    """f_in: (batch, N_in) Fourier cubes -> (batch, N_out) with the blocks of transfer_mapping_grid, zero elsewhere."""
    nb = f_in.shape[0]
    cin = f_in.reshape(nb, fft_in[2], fft_in[1], fft_in[0])
    out = np.zeros((nb, fft_out[2], fft_out[1], fft_out[0]), dtype=f_in.dtype)
    for bi, bo in transfer_mapping_grid(fft_in, fft_out):
        out[:, bo[2].start:bo[2].stop, bo[1].start:bo[1].stop, bo[0].start:bo[0].stop] = \
            cin[:, bi[2].start:bi[2].stop, bi[1].start:bi[1].stop, bi[0].start:bi[0].stop]
    return out.reshape(nb, -1)


def transfer_mapping_kpt(G_in, k_in, fft_out, mapping_out, k_out):
    """(idcs_in, idcs_out) with ψ_out[idcs_out] = ψ_in[idcs_in]; k_out = k_in + ΔG."""
    dG = np.asarray(k_out) - np.asarray(k_in)
    assert np.allclose(dG, np.round(dG), atol=1e-5)
    dG = np.round(dG).astype(np.int64)
    lin = index_G_vectors(fft_out, np.asarray(G_in) - dG)
    pos = {int(m): i for i, m in enumerate(mapping_out)}
    idcs_in, idcs_out = [], []
    for i, l in enumerate(lin):
        if l >= 0 and int(l) in pos:
            idcs_in.append(i)
            idcs_out.append(pos[int(l)])
    return np.array(idcs_in, dtype=np.int64), np.array(idcs_out, dtype=np.int64)


def transfer_blochwave_kpt(psi_k, G_in, k_in, fft_out, mapping_out, k_out):
    i, o = transfer_mapping_kpt(G_in, k_in, fft_out, mapping_out, k_out)
    out = np.zeros((len(mapping_out), psi_k.shape[1]), dtype=complex)
    out[o] = psi_k[i]
    return out


def apply_symop(S, tau, k, fft_size, G_k, psi_k, G_Sk):
    """ψSk[ig] = exp(-2πi G_full·τ) ψk[index of S⁻¹ G_full in k's sphere], G_full = G_Sk[ig] + kshift."""
    S = np.asarray(S)
    Sk_raw = S @ np.asarray(k, dtype=float)
    kshift = np.rint(normalize_kpoint_coordinate(Sk_raw) - Sk_raw).astype(np.int64)
    invS = np.rint(np.linalg.inv(S)).astype(np.int64)
    pos = {tuple(g): i for i, g in enumerate(np.asarray(G_k))}
    out = np.zeros((len(G_Sk), psi_k.shape[1]), dtype=complex)
    for ig, G in enumerate(np.asarray(G_Sk)):
        Gf = G + kshift
        src = pos[tuple(invS @ Gf)]
        out[ig] = np.exp(-2j * math.pi * float(Gf @ np.asarray(tau))) * psi_k[src]
    return out


def cell_to_supercell(psi, G_list, kcoords, kgrid, G_super):
    """ψ[k] (n_G_k, n_bands) -> one (n_G_super, n_k n_bands) block: column k n_bands + n holds ψ[k][:, n] on the rows of the
    supercell G = diag(kgrid)(G + k)."""
    pos = {tuple(g): i for i, g in enumerate(np.asarray(G_super))}
    s = np.asarray(kgrid)
    blocks = []
    for p, G, k in zip(psi, G_list, kcoords):
        b = np.zeros((len(G_super), p.shape[1]), dtype=complex)
        rows = [pos[tuple(np.rint(s * (g + np.asarray(k))).astype(np.int64))] for g in np.asarray(G)]
        b[rows] = p
        blocks.append(b)
    return np.hstack(blocks)


def bspline_coefficients(f):
    """Periodic quadratic B-spline coefficients of samples f[z, y, x]: solve (1/8, 3/4, 1/8) circulant systems per axis."""
    c = f.astype(float)
    for ax in range(3):
        n = c.shape[ax]
        A = np.zeros((n, n))
        for i in range(n):
            A[i, i] += 0.75
            A[i, (i - 1) % n] += 0.125
            A[i, (i + 1) % n] += 0.125
        c = np.moveaxis(np.tensordot(np.linalg.inv(A), np.moveaxis(c, ax, 0), axes=(1, 0)), 0, ax)
    return c


def bspline_evaluate(c, points):
    """Spline with coefficients c[z, y, x] at points (n, 3) given as (x, y, z) in units of the grid (periodic)."""
    nz, ny, nx = c.shape
    points = np.asarray(points, dtype=float)
    w, q = [], []
    for ax in range(3):
        qi = np.floor(points[:, ax] + 0.5).astype(np.int64)
        t = points[:, ax] - qi
        w.append((0.5 * (0.5 - t) ** 2, 0.75 - t * t, 0.5 * (0.5 + t) ** 2))
        q.append(qi)
    out = np.zeros(len(points))
    for a in range(3):
        for b in range(3):
            for d in range(3):
                out += w[0][a] * w[1][b] * w[2][d] * c[(q[2] + d - 1) % nz, (q[1] + b - 1) % ny, (q[0] + a - 1) % nx]
    return out


def interpolate_density(f, grid_out, rep=(1, 1, 1)):
    """f[z, y, x] on grid_in -> the output cube [z', y', x'] of a cell of rep input cells (interpolation.jl:25-89)."""
    grid_in = (f.shape[2], f.shape[1], f.shape[0])
    tiled = tuple(n * r for n, r in zip(grid_in, rep))
    if tiled == tuple(grid_out):
        return np.tile(f, (rep[2], rep[1], rep[0]))
    c = bspline_coefficients(f)
    nxo, nyo, nzo = grid_out
    Z, Y, X = np.meshgrid(np.arange(nzo), np.arange(nyo), np.arange(nxo), indexing="ij")
    pts = np.stack([X.ravel() * tiled[0] / nxo, Y.ravel() * tiled[1] / nyo, Z.ravel() * tiled[2] / nzo], axis=1)
    return bspline_evaluate(c, pts).reshape(nzo, nyo, nxo)
