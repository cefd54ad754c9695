"""Pseudopotentials for the host-side setup: analytic GTH/HGH (mirror of src/pseudo/PspHgh.jl), numerical
norm-conserving UPF (src/pseudo/PspUpf.jl) and src/elements.jl ElementPsp.  Setup code: runs once per basis,
vectorised with torch on the device; the UPF radial transforms are a CUDA kernel."""
import math
import os
import re
import numpy as np
import torch

# published GTH parameters (same numbers as the reference's data/psp/hgh/{lda,pbe}/*.hgh files)
_TABLE = {
    ("Si", "lda"): (14, [2, 2], 0.44, [-7.33610297],
                    [(0.42273813, [[5.90692831, -1.26189397], [3.25819622]]), (0.48427842, [[2.72701346]])]),
    ("Si", "pbe"): (14, [2, 2], 0.44, [-6.26928833],
                    [(0.43563383, [[8.95174150, -2.70627082], [3.49378060]]), (0.49794218, [[2.43127673]])]),
    ("Al", "lda"): (13, [2, 1], 0.45, [-8.49135116],
                    [(0.46010427, [[5.08833953, -1.03784325], [2.67969975]]), (0.53674439, [[2.19343827]])]),
    ("Al", "pbe"): (13, [2, 1], 0.45, [-7.55476126],
                    [(0.48743529, [[6.95993832, -1.88883584], [2.43847659]]), (0.56218949, [[1.86529857]])]),
    ("Fe", "pbe"): (26, [4, 6, 6], 0.36, [6.75678916, -0.22883251],
                    [(0.27826303, [[0.62950570, 7.91313242], [-10.21581002]]),
                     (0.25138338, [[-7.93213293, 7.69707888], [-9.10730654]]),
                     (0.22285578, [[-12.38579937]])]),
}
_ATOMIC_NUMBER = {"H": 1, "He": 2, "Li": 3, "C": 6, "N": 7, "O": 8, "Na": 11, "Mg": 12, "Al": 13, "Si": 14,
                  "Fe": 26, "Cu": 29, "Tl": 81}


class PspHgh:
    def __init__(self, Zion, rloc, cloc, rp, h, identifier=""):
        if len(rp) != len(h):
            raise ValueError("Length of rp and h do not agree.")
        if len(cloc) > 4:
            raise ValueError("length(cloc) > 4 not supported.")
        self.Zion, self.rloc = int(Zion), float(rloc)
        self.cloc = list(cloc) + [0.0] * (4 - len(cloc))
        self.lmax = len(h) - 1
        self.rp = [float(r) for r in rp]
        self.h = [np.array(x, dtype=float) for x in h]
        self.identifier = identifier

    def count_n_proj_radial(self, l):
        return self.h[l].shape[0]

    def count_n_proj(self):
        return sum((2 * l + 1) * self.h[l].shape[0] for l in range(self.lmax + 1))

    def count_n_pswfc_radial(self, l=None):
        """NormConservingPsp.jl:236: analytic HGH pseudopotentials carry no pseudo-atomic orbitals."""
        raise ValueError(f"Pseudopotential {self.identifier} does not implement atomic wavefunctions.")

    count_n_pswfc = count_n_pswfc_radial

    def eval_psp_local_fourier(self, p):
        """p: torch tensor of |G| values.  PspHgh.jl:110-124."""
        t = p * self.rloc
        t2 = t * t
        c = self.cloc
        poly = c[0] + c[1] * (3 - t2) + c[2] * (15 - 10 * t2 + t2 ** 2) + c[3] * (105 - 105 * t2 + 21 * t2 ** 2 - t2 ** 3)
        safe = torch.where(t2 == 0, torch.ones_like(t2), t2)
        val = (4 * math.pi * self.rloc ** 2 * (-self.Zion + math.sqrt(math.pi / 2) * self.rloc * t2 * poly)
               * torch.exp(-t2 / 2) / safe)
        return torch.where(p == 0, torch.zeros_like(val), val)

    def eval_psp_projector_fourier(self, i, l, p):
        """PspHgh.jl:140-164 (divided by p^l)."""
        rp = self.rp[l]
        t2 = (p * rp) ** 2
        common = 4 * math.pi ** 1.25 * math.sqrt(2.0 ** (l + 1) * rp ** 3) * torch.exp(-t2 / 2)
        key = (l, i)
        if key == (0, 1): return common
        if key == (0, 2): return common * (2 / math.sqrt(15)) * (3 - t2)
        if key == (0, 3): return common * (4 / (3 * math.sqrt(105))) * (15 - 10 * t2 + t2 ** 2)
        if key == (1, 1): return common * (rp / math.sqrt(3))
        if key == (1, 2): return common * (2 * rp / math.sqrt(105)) * (5 - t2)
        if key == (1, 3): return common * (4 * rp / (3 * math.sqrt(1155))) * (35 - 14 * t2 + t2 ** 2)
        if key == (2, 1): return common * (rp ** 2 / math.sqrt(15))
        if key == (2, 2): return common * (2 * rp ** 2 / (3 * math.sqrt(105))) * (7 - t2)
        if key == (3, 1): return common * (rp ** 3 / math.sqrt(105))
        raise NotImplementedError(f"Not implemented for l={l} and i={i}")

    def eval_psp_energy_correction(self):
        cc = [1.0, 3.0, 15.0, 105.0]
        dc = self.Zion * self.rloc ** 2 / 2 + math.sqrt(math.pi / 2) * self.rloc ** 3 * sum(a * b for a, b in zip(cc, self.cloc))
        return 4 * math.pi * dc


def parse_hgh(text, identifier=""):
    """The ABINIT/CP2K text format read by PspHgh(path), PspHgh.jl:25-93."""
    lines = text.splitlines()
    n_elec = [int(x) for x in re.match(r"^ *(([0-9]+ *)+)", lines[1]).group(1).split()]
    m = re.match(r"^ *([-.0-9]+) +([0-9]+)( +([-.0-9]+ *)+)? *", lines[2])
    rloc, nloc = float(m.group(1)), int(m.group(2))
    cloc = [float(x) for x in m.group(3).split()] if m.group(3) else []
    if len(cloc) != nloc:
        raise ValueError("inconsistent local coefficients")
    lmax = int(re.match(r"^ *([0-9]+)", lines[3]).group(1)) - 1
    cur, rp, h = 4, [], []
    for _ in range(lmax + 1):
        m = re.match(r"^ *([-.0-9]+) +([0-9]+)( +([-.0-9]+ *)+)? *", lines[cur])
        rp.append(float(m.group(1)))
        nproj = int(m.group(2))
        hm = np.zeros((nproj, nproj))
        if nproj == 0:
            h.append(hm)
            cur += 1
            continue
        coeff = [float(x) for x in m.group(3).split()]
        for i in range(nproj):
            for j in range(i, nproj):
                hm[i, j] = hm[j, i] = coeff[j - i]
            cur += 1
            if cur >= len(lines):
                break
            mm = re.match(r"^ *(([-.0-9]+ *)+)", lines[cur])
            coeff = [float(x) for x in mm.group(1).split()] if mm else []
        h.append(hm)
    return PspHgh(sum(n_elec), rloc, cloc, rp, h, identifier)


def _simpson_weights(x, uniform):
    """Quadrature weights of src/common/quadrature.jl (simpson_uniform / simpson_nonuniform, with the end correction for an
    odd number of intervals; trapezoidal below five points) on the nodes x."""
    n = len(x)
    w = np.zeros(n)
    if n == 1:
        return w
    if n <= 4 or uniform is None:
        w[0] = (x[1] - x[0]) / 2
        w[1:n - 1] = (x[2:] - x[:n - 2]) / 2
        w[n - 1] += (x[n - 1] - x[n - 2]) / 2
        return w
    odd = (n - 1) % 2 == 1
    if uniform:
        dx = x[1] - x[0]
        istop = n - 2 if odd else n - 1                   # last node (1-based) of the composite part
        w[0] = dx / 3
        w[1:istop:2] = 4 / 3 * dx                          # 1-based even nodes
        w[2:istop:2] = 2 / 3 * dx
        if odd:
            w[n - 1] += 5 / 12 * dx
            w[n - 2] += dx
            w[n - 3] -= dx / 12
        else:
            w[n - 1] += dx / 3
        return w
    m = n - 1 if odd else n                               # composite panels over the first m nodes
    dx0, dx1 = x[1:m:2] - x[0:m - 1:2], x[2:m:2] - x[1:m - 1:2]
    c = (dx0 + dx1) / 6
    np.add.at(w, np.arange(0, m - 2, 2), c * (2 - dx1 / dx0))
    np.add.at(w, np.arange(1, m - 1, 2), c * (dx0 + dx1) ** 2 / (dx0 * dx1))
    np.add.at(w, np.arange(2, m, 2), c * (2 - dx0 / dx1))
    if odd:
        dxn, dxm = x[-1] - x[-2], x[-2] - x[-3]
        w[n - 1] += (2 * dxn ** 2 + 3 * dxn * dxm) / (6 * (dxm + dxn))
        w[n - 2] += (dxn ** 2 + 3 * dxn * dxm) / (6 * dxm)
        w[n - 3] -= dxn ** 3 / (6 * dxm * (dxm + dxn))
    return w


class PspUpf:
    """Numerical norm-conserving pseudopotential read from a UPF v2 file (src/pseudo/PspUpf.jl).  Stored as in the
    reference: vloc in Ha, r²β per projector cut at its cutoff_radius_index, h[l] = 2·PP_DIJ, r²ρion = PP_RHOATOM/4π,
    r²ρcore = r²·PP_NLCC.  The Fourier-space form factors are radial transforms evaluated on the device
    (dftk_b200_radial_transform), once per distinct |q| of a call."""

    def __init__(self, Zion, lmax, rgrid, vloc, r2_projs, h, r2_rhoion, r2_rhocore, r2_taucore, identifier="",
                 description="", r2_pswfcs=None, pswfc_labels=None, pswfc_occs=None):
        self.Zion, self.lmax = int(Zion), int(lmax)
        self.rgrid = np.ascontiguousarray(rgrid, dtype=np.float64)
        self.vloc = np.asarray(vloc, dtype=np.float64)
        self.r2_projs = [[np.asarray(f, dtype=np.float64) for f in fl] for fl in r2_projs]
        self.h = [np.array(x, dtype=float) for x in h]
        self.r2_rhoion = np.asarray(r2_rhoion, dtype=np.float64)
        self.r2_rhocore = np.asarray(r2_rhocore, dtype=np.float64)
        self.r2_taucore = np.asarray(r2_taucore, dtype=np.float64)     # read and kept; meta-GGA is not supported
        self.rcut = float(self.rgrid[-1])
        self.identifier, self.description = identifier, description
        # pseudo-atomic orbitals r²χ per l <= lmax (PP_PSWFC, PspUpf.jl:140-155), with their labels and occupations
        self.r2_pswfcs = [[np.asarray(f, dtype=np.float64) for f in fl] for fl in (r2_pswfcs or [[]] * (self.lmax + 1))]
        self.pswfc_labels = [list(x) for x in (pswfc_labels or [[]] * (self.lmax + 1))]
        self.pswfc_occs = [list(x) for x in (pswfc_occs or [[]] * (self.lmax + 1))]
        # default_psp_quadrature: the rule is chosen on the full mesh, (x2-x1) ≈ (x3-x2) with Julia's rtol √eps, atol 0
        r = self.rgrid
        if len(r) <= 4:
            self._uniform = None
        else:
            a, b = r[1] - r[0], r[2] - r[1]
            self._uniform = bool(abs(a - b) <= math.sqrt(np.finfo(float).eps) * max(abs(a), abs(b)))
        self._tables = {}
        self._cache = (None, None)

    def count_n_proj_radial(self, l):
        return self.h[l].shape[0]

    def count_n_proj(self):
        return sum((2 * l + 1) * self.h[l].shape[0] for l in range(self.lmax + 1))

    def count_n_pswfc_radial(self, l=None):
        """Radial pseudo-atomic orbitals of angular momentum l, or of all l (NormConservingPsp.jl:238-240)."""
        if l is None:
            return sum(self.count_n_pswfc_radial(ll) for ll in range(self.lmax + 1))
        return len(self.r2_pswfcs[l])

    def count_n_pswfc(self, l=None):
        """Orbitals including their 2l+1 angular parts (NormConservingPsp.jl:242-245)."""
        if l is None:
            return sum(self.count_n_pswfc(ll) for ll in range(self.lmax + 1))
        return self.count_n_pswfc_radial(l) * (2 * l + 1)

    def pswfc_label(self, i, l):
        """Label (e.g. "3D") of the i-th (1-based) radial orbital of angular momentum l."""
        return self.pswfc_labels[l][i - 1]

    def find_pswfc(self, label):
        """(l, i) of the orbital with this label, i 1-based (NormConservingPsp.jl:247-255)."""
        for l in range(self.lmax + 1):
            for i in range(1, self.count_n_pswfc_radial(l) + 1):
                if self.pswfc_label(i, l) == label:
                    return l, i
        raise ValueError(f"Could not find pseudo atomic orbital with label {label} in pseudopotential {self.identifier}.")

    @property
    def has_core_density(self):
        return bool(np.any(self.r2_rhocore != 0))

    @property
    def has_valence_density(self):
        return bool(np.any(self.r2_rhoion != 0))

    def weights(self, n):
        """Quadrature weights of the first n mesh points (each function is integrated over its own length)."""
        return _simpson_weights(self.rgrid[:n], self._uniform)

    def _table(self, kind, device):
        """(r, g, l) on the device for one group of functions: g = weights · r²f, zero-padded to the mesh length."""
        key = (kind, str(device))
        if key not in self._tables:
            r, n = self.rgrid, len(self.rgrid)
            if kind == "proj":
                rows, ls = [], []
                for l in range(self.lmax + 1):
                    for f in self.r2_projs[l]:
                        g = np.zeros(n)
                        g[:len(f)] = self.weights(len(f)) * f
                        rows.append(g)
                        ls.append(l)
            elif kind == "pswfc":        # the orbitals are not cut off: whole mesh, whole-mesh weights (PspUpf.jl:218-223)
                rows, ls = [], []
                for l in range(self.lmax + 1):
                    for f in self.r2_pswfcs[l]:
                        rows.append(self.weights(n) * f)
                        ls.append(l)
            elif kind == "local":        # l = 0 transform of r²(vloc + Z erf(r)/r): the smooth part of PspUpf.jl:229-242
                rows, ls = [self.weights(n) * r * (r * self.vloc + self.Zion * _erf(r))], [0]
            elif kind == "core":
                rows, ls = [self.weights(n) * self.r2_rhocore], [0]
            elif kind == "valence":
                rows, ls = [self.weights(n) * self.r2_rhoion], [0]
            g = torch.from_numpy(np.ascontiguousarray(np.array(rows).reshape(len(rows), n))).to(device)
            self._tables[key] = (torch.from_numpy(r).to(device), g, np.ascontiguousarray(ls, dtype=np.int32))
        return self._tables[key]

    def radial_transform(self, kind, p):
        """F[f, :] for every function of `kind` at the |q| values p (torch, float64): the kernel runs on the distinct
        values only and the result is gathered back."""
        from ._lib import lib, check
        from .device import _ptr
        r, g, ls = self._table(kind, p.device)
        flat = p.reshape(-1).contiguous()
        uq, inv = torch.unique(flat, return_inverse=True)
        uq = uq.contiguous()
        F = torch.empty((len(ls), uq.numel()), dtype=torch.float64, device=p.device)
        h = _radial_ctx(p.device)
        check(lib().dftk_b200_radial_transform(h, len(r), _ptr(r), len(ls), _ptr(g), _ptr(ls), uq.numel(), _ptr(uq), _ptr(F)), h)
        return F[:, inv].reshape((len(ls),) + tuple(p.shape))

    def eval_psp_projector_fourier(self, i, l, p):
        # build_projector_form_factors asks for every (l, i) at the same |G+k|: one launch serves all projectors of the
        # pseudopotential, and the rows are kept while the caller holds on to that tensor
        if self._cache[0] is not p:
            self._cache = (p, self.radial_transform("proj", p))
        row = sum(self.count_n_proj_radial(ll) for ll in range(l)) + i - 1
        return self._cache[1][row]

    def eval_psp_pswfc_fourier(self, i, l, p):
        """Radial part of the i-th (1-based) orbital of angular momentum l at |q| = p, divided by p^l like the projectors;
        one launch serves all orbitals while the caller holds on to p."""
        if getattr(self, "_pswfc_cache", (None,))[0] is not p:
            self._pswfc_cache = (p, self.radial_transform("pswfc", p))
        return self._pswfc_cache[1][sum(self.count_n_pswfc_radial(ll) for ll in range(l)) + i - 1]

    def eval_psp_local_fourier(self, p):
        F = self.radial_transform("local", p)[0]
        safe = torch.where(p == 0, torch.ones_like(p), p)
        F = F - 4 * math.pi * self.Zion * torch.exp(-safe * safe / 4) / (safe * safe)
        return torch.where(p == 0, torch.zeros_like(F), F)

    def eval_psp_core_density_fourier(self, p):
        return self.radial_transform("core", p)[0]

    def eval_psp_valence_density_fourier(self, p):
        return self.radial_transform("valence", p)[0]

    def eval_psp_energy_correction(self):
        r = self.rgrid
        return 4 * math.pi * float(np.sum(self.weights(len(r)) * r * (r * self.vloc + self.Zion)))


def _erf(x):
    from scipy.special import erf
    return erf(x)


def _radial_ctx(device):
    """The library context of the GPU that holds p: the one a basis on that device already uses, else the context
    B200(device) would create."""
    from .architecture import B200
    idx = device.index if device.index is not None else torch.cuda.current_device()
    for c in B200._contexts.values():
        if c.device.index == idx:
            return c.h
    return B200(device=idx).ctx.h


def _upf_values(node):
    return np.array(node.text.split(), dtype=float)


def parse_upf(text, identifier=""):
    """UPF v2 (XML) reader with the unit conversions of PspUpf.jl:97-158."""
    import xml.etree.ElementTree as ET
    if not re.search(r"<UPF\s+version\s*=\s*\"2", text[:4096]):
        raise ValueError("UPF: only version 2 (XML) files are supported")
    root = ET.fromstring(text)
    hd = root.find("PP_HEADER")
    flag = lambda k: hd.get(k, "F").strip().upper() in ("T", "TRUE", ".TRUE.")
    ptype = hd.get("pseudo_type", "").strip()
    unsupported = []
    if flag("has_so"):
        unsupported.append("spin-orbit coupling")
    if ptype == "SL":
        unsupported.append("semilocal potential")
    if ptype in ("US", "USPP"):
        unsupported.append("ultrasoft")
    if ptype == "PAW":
        unsupported.append("projector-augmented wave")
    if flag("has_gipaw"):
        unsupported.append("gipaw data")
    if ptype == "1/r":
        unsupported.append("Coulomb")
    if unsupported:
        raise ValueError("Pseudopotential contains the following unsupported features/quantities: " + ",".join(unsupported))
    lmax = int(hd.get("l_max"))
    if lmax > 3:
        raise ValueError(f"UPF: l_max = {lmax} > 3 is not supported (solid harmonics stop at l = 3)")
    rgrid = _upf_values(root.find("PP_MESH").find("PP_R"))
    n = len(rgrid)
    vloc = _upf_values(root.find("PP_LOCAL"))[:n] / 2                   # Ry -> Ha
    nl = root.find("PP_NONLOCAL")
    betas = [b for b in nl if b.tag.startswith("PP_BETA")] if nl is not None else []
    nb = len(betas)
    dij = _upf_values(nl.find("PP_DIJ")).reshape(nb, nb) * 2 if nb else np.zeros((0, 0))    # 1/Ry -> 1/Ha
    ang = [int(b.get("angular_momentum")) for b in betas]
    r2_projs, h = [], []
    for l in range(lmax + 1):
        idx = [i for i in range(nb) if ang[i] == l]
        fl = []
        for i in idx:
            cut = int(betas[i].get("cutoff_radius_index", str(n)))
            fl.append(rgrid[:cut] * (_upf_values(betas[i])[:cut] / 2))        # rβ (Ry) -> r²β (Ha)
        r2_projs.append(fl)
        h.append(dij[np.ix_(idx, idx)])
    opt = lambda tag: root.find(tag)
    rho = opt("PP_RHOATOM")
    r2_rhoion = _upf_values(rho)[:n] / (4 * math.pi) if rho is not None else np.zeros(n)
    nlcc = opt("PP_NLCC")
    r2_rhocore = rgrid ** 2 * _upf_values(nlcc)[:n] if nlcc is not None else np.zeros(n)
    tau = opt("PP_TAUMOD")
    r2_taucore = rgrid ** 2 * _upf_values(tau)[:n] if tau is not None else np.zeros(n)
    r2_pswfcs, labels, occs = [[] for _ in range(lmax + 1)], [[] for _ in range(lmax + 1)], [[] for _ in range(lmax + 1)]
    wfc = opt("PP_PSWFC")
    for chi in ([c for c in wfc if c.tag.startswith("PP_CHI")] if wfc is not None else []):
        l = int(chi.get("l"))
        if l > lmax:
            continue
        r2_pswfcs[l].append(rgrid * _upf_values(chi)[:n])                   # rχ -> r²χ
        labels[l].append((chi.get("label") or "").strip())
        occs[l].append(float(chi.get("occupation", "0")))
    return PspUpf(round(float(hd.get("z_valence"))), lmax, rgrid, vloc, r2_projs, h, r2_rhoion, r2_rhocore, r2_taucore,
                  identifier=identifier, description=(hd.get("comment") or "").strip(), r2_pswfcs=r2_pswfcs,
                  pswfc_labels=labels, pswfc_occs=occs)


def load_psp(symbol, functional="lda"):
    """load_psp(symbol, functional): the built-in GTH tables; load_psp(path): a .upf, .hgh or .gth file."""
    ext = os.path.splitext(str(symbol))[1].lower()
    if ext in (".upf", ".hgh", ".gth"):
        with open(symbol) as fh:
            text = fh.read()
        return parse_upf(text, identifier=str(symbol)) if ext == ".upf" else parse_hgh(text, identifier=str(symbol))
    Z, n_elec, rloc, cloc, proj = _TABLE[(symbol, functional)]
    rp, h = [], []
    for r, rows in proj:
        n = len(rows)
        hm = np.zeros((n, n))
        for i, row in enumerate(rows):
            for j, v in enumerate(row):
                hm[i, i + j] = hm[i + j, i] = v
        rp.append(r)
        h.append(hm)
    return PspHgh(sum(n_elec), rloc, cloc, rp, h, identifier=f"hgh/{functional}/{symbol.lower()}-q{sum(n_elec)}")


class ElementPsp:
    """src/elements.jl ElementPsp: species + pseudopotential."""

    def __init__(self, symbol, psp=None, functional="lda"):
        self.symbol = symbol
        self.Z = _ATOMIC_NUMBER[symbol]
        self.psp = psp if psp is not None else load_psp(symbol, functional)

    def charge_ionic(self):
        return self.psp.Zion

    def n_elec_valence(self):
        return self.psp.Zion

    def n_elec_core(self):
        return self.Z - self.psp.Zion

    def __eq__(self, o):
        return isinstance(o, ElementPsp) and o.symbol == self.symbol and o.psp.identifier == self.psp.identifier

    def __hash__(self):
        return hash((self.symbol, self.psp.identifier))


def atom_decay_length(n_elec_core, n_elec_valence):
    """density_methods.jl:286-323 (ABINIT table)."""
    nv = int(round(n_elec_valence))
    if nv == 0:
        return 0.0
    tables = [(0.5, [0.6, 0.4, 0.3, 0.25, 0.2]),
              (2.5, [1.8, 1.4, 1.0, 0.7, 0.6, 0.5, 0.4, 0.35, 0.3]),
              (10.5, [2.0, 1.6, 1.25, 1.1, 1.0, 0.9, 0.8, 0.7, 0.7, 0.7, 0.6]),
              (12.5, [1.9, 1.5, 1.15, 1.0, 0.9, 0.8, 0.7, 0.6, 0.6, 0.6, 0.5]),
              (18.5, [2.0, 1.8, 1.5, 1.2, 1.0, 0.9, 0.85, 0.8, 0.75, 0.7, 0.65, 0.65, 0.6]),
              (28.5, [1.5, 1.25, 1.15, 1.05, 1.00, 0.95, 0.95, 0.9, 0.9, 0.85, 0.85, 0.80, 0.8, 0.75, 0.7]),
              (36.5, [2.0, 2.00, 1.60, 1.40, 1.25, 1.10, 1.00, 0.95, 0.90, 0.85, 0.80, 0.75, 0.7])]
    data = [2.0, 2.00, 1.55, 1.25, 1.15, 1.10, 1.05, 1.0, 0.95, 0.9, 0.85, 0.85, 0.8]
    for lim, d in tables:
        if n_elec_core < lim:
            data = d
            break
    return data[min(nv, len(data)) - 1]


def solid_harmonic_real(l, m, v):
    """Real solid harmonics on a (n,3) torch tensor (src/common/spherical_harmonics.jl:31-66)."""
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    pi = math.pi
    if l == 0:
        return torch.full_like(x, math.sqrt(1 / (4 * pi)))
    if l == 1:
        return math.sqrt(3 / (4 * pi)) * {-1: y, 0: z, 1: x}[m]
    if l == 2:
        return {-2: math.sqrt(15 / (4 * pi)) * x * y, -1: math.sqrt(15 / (4 * pi)) * y * z,
                0: math.sqrt(5 / (16 * pi)) * (2 * z * z - x * x - y * y),
                1: math.sqrt(15 / (4 * pi)) * x * z, 2: math.sqrt(15 / (16 * pi)) * (x * x - y * y)}[m]
    if l == 3:
        return {-3: math.sqrt(35 / (32 * pi)) * (3 * x * x - y * y) * y,
                -2: math.sqrt(105 / (4 * pi)) * x * y * z,
                -1: math.sqrt(21 / (32 * pi)) * y * (4 * z * z - x * x - y * y),
                0: math.sqrt(7 / (16 * pi)) * z * (2 * z * z - 3 * x * x - 3 * y * y),
                1: math.sqrt(21 / (32 * pi)) * x * (4 * z * z - x * x - y * y),
                2: math.sqrt(105 / (16 * pi)) * (x * x - y * y) * z,
                3: math.sqrt(35 / (32 * pi)) * (x * x - 3 * y * y) * x}[m]
    raise IndexError((l, m))
