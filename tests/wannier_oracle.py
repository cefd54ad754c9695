"""Independent NumPy restatement of the Wannier90 interface (reference: src/external/wannier_shared.jl,
src/common/hydrogenic.jl), written literally: common G vectors searched one at a time, one dot product per matrix entry.
Plus, for tests only, the b-vectors of a Monkhorst-Pack mesh as Wannier90's kmesh step finds them (the package takes them
from `wannier90.x -pp`)."""
import math

import numpy as np
from scipy.special import spherical_jn


# ------------------------------------------------------------------ matrices
def overlap_Mmn_k_kpb(G_k, psi_k, G_kpb, psi_kpb, G_shift, n_bands):
    """wannier_shared.jl:220-241.  G_*: (n_G, 3) integer G vectors of each sphere, psi_*: (n_bands_total, n_G)."""
    where = {tuple(int(x) for x in g): i for i, g in enumerate(G_kpb)}
    ip, ip_plus_b = [], []
    for i, g in enumerate(G_k):
        j = where.get(tuple(int(x) + int(s) for x, s in zip(g, G_shift)))
        if j is not None:
            ip.append(i)
            ip_plus_b.append(j)
    M = np.zeros((n_bands, n_bands), dtype=complex)
    for n in range(n_bands):
        for m in range(n_bands):
            M[m, n] = np.vdot(psi_k[m, ip], psi_kpb[n, ip_plus_b])
    if not M.any():
        return np.eye(n_bands, dtype=complex)
    return M


def compute_amn_kpoint(psi_k, gn, n_bands):
    """wannier_shared.jl:278-298 with the projection values gn (n_wannier, n_G) already evaluated."""
    A = np.zeros((n_bands, len(gn)), dtype=complex)
    for n, g in enumerate(gn):
        c = g / np.linalg.norm(g)
        for m in range(n_bands):
            A[m, n] = np.vdot(psi_k[m], c)
    return A


# ------------------------------------------------------------------ projections
def gaussian(ps, recip, center):
    pc = ps @ recip.T
    return np.exp(2 * np.pi * (-1j * (ps @ center) - np.sum(pc * pc, axis=1) / 4))


def radial_hydrogenic(r, n, alpha=1.0):
    if n == 1:
        return 2 * alpha ** 1.5 * np.exp(-alpha * r)
    if n == 2:
        return 2 ** -1.5 * alpha ** 1.5 * (2 - alpha * r) * np.exp(-alpha * r / 2)
    if n == 3:
        return np.sqrt(4 / 27) * alpha ** 1.5 * (1 - 2 / 3 * alpha * r + 2 / 27 * alpha ** 2 * r ** 2) * np.exp(-alpha * r / 3)
    raise ValueError(n)


def ylm_real(l, m, v):
    """Real spherical harmonics of the direction of each row of v (src/common/spherical_harmonics.jl), 0 at v = 0 for l > 0."""
    nrm = np.linalg.norm(v, axis=1)
    safe = np.where(nrm > 0, nrm, 1.0)
    x, y, z = v[:, 0] / safe, v[:, 1] / safe, v[:, 2] / safe
    if l == 0:
        return np.full(len(v), np.sqrt(1 / (4 * np.pi)))
    table = {
        (1, -1): np.sqrt(3 / (4 * np.pi)) * y, (1, 0): np.sqrt(3 / (4 * np.pi)) * z, (1, 1): np.sqrt(3 / (4 * np.pi)) * x,
        (2, -2): np.sqrt(15 / (4 * np.pi)) * x * y, (2, -1): np.sqrt(15 / (4 * np.pi)) * y * z,
        (2, 0): np.sqrt(5 / (16 * np.pi)) * (3 * z * z - 1), (2, 1): np.sqrt(15 / (4 * np.pi)) * x * z,
        (2, 2): np.sqrt(15 / (16 * np.pi)) * (x * x - y * y),
        (3, -3): np.sqrt(35 / (32 * np.pi)) * (3 * x * x - y * y) * y, (3, -2): np.sqrt(105 / (4 * np.pi)) * x * y * z,
        (3, -1): np.sqrt(21 / (32 * np.pi)) * y * (5 * z * z - 1), (3, 0): np.sqrt(7 / (16 * np.pi)) * z * (5 * z * z - 3),
        (3, 1): np.sqrt(21 / (32 * np.pi)) * x * (5 * z * z - 1), (3, 2): np.sqrt(105 / (16 * np.pi)) * (x * x - y * y) * z,
        (3, 3): np.sqrt(35 / (32 * np.pi)) * (x * x - 3 * y * y) * x}
    return np.where(nrm > 0, table[(l, m)], 0.0)


def hydrogenic(ps, recip, center, n, l, m, alpha):
    """wannier_shared.jl:37-71, without the 4π as in the reference."""
    xmin, dx, rmax = -6.0, 0.025, 10.0
    n_r = int(round((math.log(rmax) - xmin) / dx)) + 1
    r = np.exp(xmin + dx * np.arange(n_r)) / alpha
    r2_R_dr = r ** 2 * radial_hydrogenic(r, n, alpha) * r * dx
    pc = ps @ recip.T
    pn = np.linalg.norm(pc, axis=1)
    radial = np.array([np.sum(r2_R_dr * spherical_jn(l, q * r)) for q in pn])
    return np.exp(-2j * np.pi * (ps @ center)) * ylm_real(l, m, pc) * (-1j) ** l * radial


# ------------------------------------------------------------------ files
def unk(cube_shape, mapping, psi_kn, volume):
    """ifft(basis, kpt, ψ) of one band: the periodic part on the real-space grid, x fastest (flattened)."""
    nx, ny, nz = cube_shape
    c = np.zeros(nx * ny * nz, dtype=complex)
    c[mapping] = psi_kn
    return np.fft.ifftn(c.reshape(nz, ny, nx)).reshape(-1) * (nx * ny * nz) / np.sqrt(volume)


def write_nnkp(path, nntot, nnkpts):
    """The nnkpts block of a .nnkp file (1-based k-point indices)."""
    with open(path, "w") as fp:
        fp.write("File written by the test b-vector helper\n\nbegin nnkpts\n")
        fp.write(f"{nntot:4d}\n")
        for ik, ikb, G in nnkpts:
            fp.write("%6d %6d %4d %4d %4d\n" % (ik + 1, ikb + 1, G[0], G[1], G[2]))
        fp.write("end nnkpts\n")


# ------------------------------------------------------------------ b-vectors (tests only)
def bvector_shells(recip, kgrid, n_max=3, tol=1e-8):
    """Shells of mesh vectors b = recip (n / kgrid), n integer, in order of length, each a list of reduced b."""
    ks = np.asarray(kgrid, dtype=float)
    rng = range(-n_max, n_max + 1)
    vecs = [np.array([i, j, k]) / ks for i in rng for j in rng for k in rng if (i, j, k) != (0, 0, 0)]
    lens = [np.linalg.norm(recip @ b) for b in vecs]
    order = np.argsort(lens, kind="stable")
    shells, cur, cur_len = [], [], None
    for i in order:
        if cur_len is not None and lens[i] - cur_len > tol * cur_len:
            shells.append(cur)
            cur = []
        if not cur:
            cur_len = lens[i]
        cur.append(vecs[i])
    shells.append(cur)
    return shells


def bvectors(recip, kgrid, max_shells=6):
    """Shells added in order of length until Σ_b w_b b bᵀ = I holds (least squares on the six components, residual < 1e-10):
    (list of reduced b, list of Cartesian b, list of weights)."""
    comps = [(0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 2)]
    rhs = np.array([1, 1, 1, 0, 0, 0], dtype=float)
    shells = bvector_shells(recip, kgrid)
    for n in range(1, max_shells + 1):
        cols = []
        for sh in shells[:n]:
            bc = np.array([recip @ b for b in sh])
            cols.append([np.sum(bc[:, a] * bc[:, c]) for a, c in comps])
        Amat = np.array(cols).T
        w, *_ = np.linalg.lstsq(Amat, rhs, rcond=None)
        if np.linalg.norm(Amat @ w - rhs) < 1e-10:
            red = [b for sh in shells[:n] for b in sh]
            weights = [w[s] for s, sh in enumerate(shells[:n]) for _ in sh]
            return red, [recip @ b for b in red], weights
    raise ValueError("no set of shells satisfies the B1 condition")


def nnkp_list(kcoords, recip, kgrid):
    """(nntot, [(ik, ik_plus_b, G_shift)], weights, Cartesian b): for every k-point and b, the k-point equal to k + b up to
    the integer vector G_shift = k + b - k_{ik_plus_b}.  0-based."""
    red, cart, w = bvectors(recip, kgrid)
    kc = np.asarray(kcoords, dtype=float)
    out = []
    for ik, k in enumerate(kc):
        for b in red:
            t = k + b
            d = t[None, :] - kc
            hit = np.nonzero(np.all(np.abs(d - np.round(d)) < 1e-8, axis=1))[0]
            assert len(hit) == 1
            j = int(hit[0])
            out.append((ik, j, tuple(int(x) for x in np.round(t - kc[j]))))
    return len(red), out, w, cart
