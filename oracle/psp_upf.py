"""Norm-conserving UPF pseudopotentials (oracle; test infrastructure only).

Follows src/pseudo/PspUpf.jl:97-260, src/common/hankel.jl and src/common/quadrature.jl of the reference.  The
spherical Bessel functions come from scipy.special.spherical_jn, so nothing here shares a formula with the device
kernel.  Only UPF v2 (XML) files with a norm-conserving, scalar-relativistic pseudopotential are read.
"""
import math
import re
import xml.etree.ElementTree as ET
import numpy as np
from scipy.special import erf, spherical_jn

ATOMIC_NUMBER = {"H": 1, "He": 2, "Li": 3, "C": 6, "N": 7, "O": 8, "Na": 11, "Mg": 12, "Al": 13, "Si": 14, "Fe": 26,
                 "Cu": 29, "Tl": 81}


def _values(node):
    return np.array(node.text.split(), dtype=float)


def _flag(header, key):
    return header.get(key, "F").strip().upper() in ("T", "TRUE", ".TRUE.")


# ------------------------------------------------------------------ quadrature.jl
def trapezoidal_weights(x):
    n = len(x)
    w = np.zeros(n)
    if n == 1:
        return w
    w[0] = (x[1] - x[0]) / 2
    w[1:n - 1] = (x[2:] - x[:n - 2]) / 2
    w[n - 1] += (x[n - 1] - x[n - 2]) / 2
    return w


def simpson_uniform_weights(x):
    n = len(x)
    dx = x[1] - x[0]
    odd = (n - 1) % 2 == 1
    istop = n - 2 if odd else n - 1          # 1-based, as in the reference
    w = np.zeros(n)
    w[0] = dx / 3
    for i in range(2, istop + 1):             # 1-based i
        w[i - 1] += (4 / 3 if i % 2 == 0 else 2 / 3) * dx
    if odd:
        w[n - 1] += 5 / 12 * dx
        w[n - 2] += dx
        w[n - 3] -= 1 / 12 * dx
    else:
        w[n - 1] += dx / 3
    return w


def simpson_nonuniform_weights(x):
    n = len(x)
    odd = (n - 1) % 2 == 1
    istop = n - 3 if odd else n - 2           # 1-based
    w = np.zeros(n)
    for i in range(1, istop + 1, 2):
        a, b, c = i - 1, i, i + 1
        dx0, dx1 = x[b] - x[a], x[c] - x[b]
        cc = (dx0 + dx1) / 6
        w[a] += cc * (2 - dx1 / dx0)
        w[b] += cc * (dx0 + dx1) ** 2 / (dx0 * dx1)
        w[c] += cc * (2 - dx0 / dx1)
    if odd:
        dxn, dxm = x[-1] - x[-2], x[-2] - x[-3]
        w[n - 1] += (2 * dxn ** 2 + 3 * dxn * dxm) / (6 * (dxm + dxn))
        w[n - 2] += (dxn ** 2 + 3 * dxn * dxm) / (6 * dxm)
        w[n - 3] -= dxn ** 3 / (6 * dxm * (dxm + dxn))
    return w


def is_uniform(x):
    """Julia's (x[2]-x[1]) ≈ (x[3]-x[2]): rtol √eps, atol 0."""
    a, b = x[1] - x[0], x[2] - x[1]
    return abs(a - b) <= math.sqrt(np.finfo(float).eps) * max(abs(a), abs(b))


def psp_quadrature_weights(full_mesh, n):
    """default_psp_quadrature(full mesh) applied to the first n points."""
    x = full_mesh[:n]
    if len(full_mesh) <= 4:
        return trapezoidal_weights(x)
    return simpson_uniform_weights(x) if is_uniform(full_mesh) else simpson_nonuniform_weights(x)


def hankel(r, r2f, l, p, w):
    """4π/p^l Σ_i w_i r2f_i j_l(p r_i); p -> 0 limit below 10 eps (hankel.jl:26-41)."""
    p = np.atleast_1d(np.asarray(p, dtype=float))
    out = np.empty(len(p))
    wf = w * r2f
    small = np.abs(p) <= 10 * np.finfo(float).eps
    dfact = [1, 3, 15, 105][l]
    out[small] = 4 * math.pi * np.sum(wf * r ** l) / dfact
    idx = np.nonzero(~small)[0]
    for c in range(0, len(idx), 256):
        pc = p[idx[c:c + 256]]
        jl = spherical_jn(l, pc[:, None] * r[None, :])
        out[idx[c:c + 256]] = 4 * math.pi * (jl @ wf) / pc ** l
    return out


class PspUpf:
    def __init__(self, text, description=""):
        if not re.search(r"<UPF\s+version\s*=\s*\"2", text[:4096]):
            raise ValueError("only UPF version 2 (XML) is supported")
        root = ET.fromstring(text)
        hd = root.find("PP_HEADER")
        bad = []
        ptype = hd.get("pseudo_type", "").strip()
        if _flag(hd, "has_so"): bad.append("spin-orbit coupling")
        if ptype == "SL": bad.append("semilocal potential")
        if ptype in ("US", "USPP"): bad.append("ultrasoft")
        if ptype == "PAW": bad.append("projector-augmented wave")
        if _flag(hd, "has_gipaw"): bad.append("gipaw data")
        if ptype == "1/r": bad.append("Coulomb")
        if bad:
            raise ValueError("unsupported: " + ",".join(bad))
        self.lmax = int(hd.get("l_max"))
        if self.lmax > 3:
            raise ValueError("l_max > 3")
        self.Zion = int(round(float(hd.get("z_valence"))))
        self.element = hd.get("element").strip()
        self.Z = ATOMIC_NUMBER[self.element]
        self.description = description or f"upf/{self.element}"
        mesh = root.find("PP_MESH")
        self.rgrid = _values(mesh.find("PP_R"))
        n = len(self.rgrid)
        self.vloc = _values(root.find("PP_LOCAL"))[:n] / 2
        nl = root.find("PP_NONLOCAL")
        betas = [b for b in nl if b.tag.startswith("PP_BETA")]
        nb = len(betas)
        dij = _values(nl.find("PP_DIJ")).reshape(nb, nb) * 2 if nb else np.zeros((0, 0))
        ls = [int(b.get("angular_momentum")) for b in betas]
        self.r2_projs, self.h = [], []
        for l in range(self.lmax + 1):
            idx = [i for i in range(nb) if ls[i] == l]
            projs = []
            for i in idx:
                cut = int(betas[i].get("cutoff_radius_index", str(n)))
                projs.append(self.rgrid[:cut] * _values(betas[i])[:cut] / 2)
            self.r2_projs.append(projs)
            self.h.append(dij[np.ix_(idx, idx)])
        rho = root.find("PP_RHOATOM")
        self.r2_rhoion = _values(rho)[:n] / (4 * math.pi) if rho is not None else np.zeros(n)
        nlcc = root.find("PP_NLCC")
        self.r2_rhocore = self.rgrid ** 2 * _values(nlcc)[:n] if nlcc is not None else np.zeros(n)

    def n_proj_radial(self, l):
        return self.h[l].shape[0]

    def n_proj(self):
        return sum((2 * l + 1) * self.n_proj_radial(l) for l in range(self.lmax + 1))

    @property
    def has_core_density(self):
        return bool(np.any(self.r2_rhocore != 0))

    @property
    def has_valence_density(self):
        return bool(np.any(self.r2_rhoion != 0))

    def _w(self, n):
        return psp_quadrature_weights(self.rgrid, n)

    def eval_projector_fourier(self, i, l, p):
        f = self.r2_projs[l][i - 1]
        return hankel(self.rgrid[:len(f)], f, l, p, self._w(len(f)))

    def eval_local_fourier(self, p):
        p = np.atleast_1d(np.asarray(p, dtype=float))
        r = self.rgrid
        f = r * (r * self.vloc + self.Zion * erf(r))            # r²·(vloc(r) + Z erf(r)/r)
        out = hankel(r, f, 0, p, self._w(len(r)))
        nz = p != 0
        out[nz] += 4 * math.pi * (-self.Zion / p[nz] ** 2 * np.exp(-p[nz] ** 2 / 4))
        out[~nz] = 0.0
        return out

    def eval_core_density_fourier(self, p):
        return hankel(self.rgrid, self.r2_rhocore, 0, p, self._w(len(self.rgrid)))

    def eval_valence_density_fourier(self, p):
        return hankel(self.rgrid, self.r2_rhoion, 0, p, self._w(len(self.rgrid)))

    def energy_correction(self):
        r = self.rgrid
        return 4 * math.pi * float(np.sum(self._w(len(r)) * r * (r * self.vloc + self.Zion)))

    # real-space forms by linear interpolation (PspUpf.jl:178-253)
    def eval_local_real(self, r):
        return np.interp(r, self.rgrid, self.vloc)

    def eval_projector_real(self, i, l, r):
        f = self.r2_projs[l][i - 1]
        return np.interp(r, self.rgrid[:len(f)], f, right=0.0) / r ** 2

    def eval_core_density_real(self, r):
        return np.interp(r, self.rgrid, self.r2_rhocore) / r ** 2

    def eval_valence_density_real(self, r):
        return np.interp(r, self.rgrid, self.r2_rhoion) / r ** 2


def load(path):
    """A .upf file, or one compressed as .upf.xz."""
    import lzma
    with (lzma.open(path, "rt") if path.endswith(".xz") else open(path)) as fh:
        return PspUpf(fh.read(), description=path)
