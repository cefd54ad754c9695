"""DFT+U: ortho-atomic orbitals and the Hubbard term (host-side mirror of src/terms/hubbard.jl,
src/postprocess/dos.jl:156-196 atomic_orbital_projectors, src/common/ortho.jl ortho_lowdin and the Hubbard parts of
src/symmetry.jl / src/common/spherical_harmonics.jl).

The orbital table Φ_k is built on the device (radial transform, dftk_b200_build_projectors, Löwdin step on the library's
GEMMs) and attached to every k-block (dftk_b200_kblock_set_orbitals): the Hubbard operator Φ V_σ Φ' then rides in the
nonlocal projector products of every H apply, and V_σ is re-installed each SCF step
(dftk_b200_kblock_set_orbital_coefficients).  The occupation matrices come from dftk_b200_orbital_occupation_multi.

Atom indices are 0-based, like every atom index of this package (the reference counts from 1).  Radial orbital indices
`i` of an `(l, i)` pair are 1-based, as in the pseudopotential API (`eval_psp_pswfc_fourier(i, l, p)`).
"""
import math
import numpy as np
import torch

from .model import SYMMETRY_TOLERANCE
from .pseudo import solid_harmonic_real


class OrbitalManifold:
    """hubbard.jl:19-28: the atoms (a species symbol, an ElementPsp, or a list of 0-based atom indices) and the orbitals
    (a label such as "3D", or an (l, i) pair with i 1-based) that carry a Hubbard correction."""

    def __init__(self, atoms, projectors):
        if hasattr(atoms, "symbol") and hasattr(atoms, "psp"):
            atoms = atoms.symbol
        if not isinstance(atoms, str):
            atoms = [int(a) for a in atoms]
        if not isinstance(projectors, str):
            l, i = projectors
            projectors = (int(l), int(i))
        self.atoms, self.projectors = atoms, projectors

    def __repr__(self):
        return f"OrbitalManifold({self.atoms!r}, {self.projectors!r})"


class ResolvedOrbitalManifold:
    def __init__(self, psp, iatoms, l, i):
        self.psp, self.iatoms, self.l, self.i = psp, list(iatoms), int(l), int(i)


def _is_approx_integer(v, atol):
    return bool(np.all(np.abs(v - np.round(v)) <= atol))


def resolve_hubbard_manifold(manifold, model):
    """hubbard.jl:44-88."""
    if isinstance(manifold.atoms, str):
        iatoms = [ia for ia, a in enumerate(model.atoms) if getattr(a, "symbol", None) == manifold.atoms]
    else:
        iatoms = list(manifold.atoms)
        if any(ia < 0 or ia >= len(model.atoms) for ia in iatoms):
            raise ValueError(f"Orbital manifold atom index out of range (0-based, {len(model.atoms)} atoms): {iatoms}")
    if not iatoms:
        raise ValueError("Orbital manifold has no atoms.")
    if any(getattr(model.atoms[ia], "psp", None) is None for ia in iatoms):
        raise ValueError("Orbital manifold elements must have a psp.")
    psp = model.atoms[iatoms[0]].psp
    for ia in iatoms:
        if model.atoms[ia].psp is not psp:
            raise ValueError(f"Orbital manifold contains multiple psps: {psp.identifier} and {model.atoms[ia].psp.identifier}")
    pos = [model.positions[ia] for ia in iatoms]
    for op in model.symmetries:
        for c in pos:
            if not any(_is_approx_integer(op.W @ c + op.w - d, SYMMETRY_TOLERANCE) for d in pos):
                raise ValueError("Inconsistency between orbital manifold and model symmetries: cannot map the atom at "
                                 f"position {c} to another atom of the manifold under the symmetry operation "
                                 f"({op.W.tolist()}, {op.w.tolist()})")
    if isinstance(manifold.projectors, str):
        l, i = psp.find_pswfc(manifold.projectors)
    else:
        l, i = manifold.projectors
    return ResolvedOrbitalManifold(psp, iatoms, l, i)


class Hubbard:
    """hubbard.jl:103-133: Hubbard([manifold, ...], [U, ...]) or Hubbard((manifold, U), ...); U in Hartree.  Passed to
    model_atomic / model_DFT in `extra_terms`; its energy is named "Hubbard"."""
    name = "Hubbard"

    def __init__(self, *args):
        if len(args) == 2 and isinstance(args[0], (list, tuple)) and all(isinstance(m, OrbitalManifold) for m in args[0]):
            manifolds, U = list(args[0]), [float(u) for u in args[1]]
        else:
            manifolds, U = [a[0] for a in args], [float(a[1]) for a in args]
        if len(manifolds) != len(U):
            raise ValueError(f"Number of U values ({len(U)}) must match number of manifolds ({len(manifolds)}).")
        self.manifolds, self.U = manifolds, U

    def __call__(self, basis):
        return TermHubbard(basis, self)


# ------------------------------------------------------------------ ortho-atomic orbitals
def _orbital_rows(psp, Gpk_cart):
    """Form factors of all orbitals of one species, ordered (l, n, m) like dos.jl:174-190: (n_rows, n_pw) complex."""
    pn = Gpk_cart.norm(dim=1)
    rows = []
    for l in range(psp.lmax + 1):
        for n in range(1, psp.count_n_pswfc_radial(l) + 1):
            radial = psp.eval_psp_pswfc_fourier(n, l, pn)
            for m in range(-l, l + 1):
                rows.append(radial * solid_harmonic_real(l, m, Gpk_cart).to(torch.complex128) * ((-1j) ** l))
    return rows


def orbital_labels(model):
    """(iatom, species, n, l, m, label) of every orbital of the complete set, in table order (dos.jl:170-191)."""
    labels = []
    for ia, atom in enumerate(model.atoms):
        psp = atom.psp
        if psp.count_n_pswfc() == 0:
            raise ValueError(f"Pseudopotential {psp.identifier} has no pseudo-atomic orbitals")
        for l in range(psp.lmax + 1):
            for n in range(1, psp.count_n_pswfc_radial(l) + 1):
                for m in range(-l, l + 1):
                    labels.append(dict(iatom=ia, species=atom.symbol, n=n, l=l, m=m, label=psp.pswfc_label(n, l)))
    return labels


def ortho_lowdin(ctx, phi):
    """common/ortho.jl ortho_lowdin on the device: phi (n_orb, n_pw) rows = orbitals.  S = Φ'Φ and Φ S^{-1/2} are
    products on the library's GEMMs; the small Hermitian eigendecomposition of S runs on the host."""
    n = phi.shape[0]
    S = torch.empty((n, n), dtype=torch.complex128, device=phi.device)
    ctx.zgemm("C", phi, phi, S)
    S = S.cpu().numpy().T                                   # column-major result -> S[i, j] = <φ_i|φ_j>
    S = (S + S.conj().T) / 2
    ev, U = np.linalg.eigh(S)
    if not np.min(np.abs(ev)) > np.finfo(float).eps * np.max(np.abs(ev)):
        raise AssertionError("ortho_lowdin: the atomic orbitals are linearly dependent")
    X = (U * ev ** -0.5) @ U.conj().T                       # S^{-1/2}
    out = torch.empty_like(phi)
    ctx.zgemm("N", phi, torch.from_numpy(np.ascontiguousarray(X.T)).to(phi.device), out)
    return out


def atomic_orbital_projectors(basis):
    """dos.jl:156-196: the Löwdin-orthonormalised pseudo-atomic orbitals of every atom, per k-point of this rank.
    Returns (projectors, labels): projectors[ik] is (n_orb, n_pw) complex on the device (a row per orbital, i.e. the
    column-major n_pw × n_orb table), labels one dict per row."""
    from ._lib import check
    from .device import _ptr
    model = basis.model
    ctx = basis.architecture.ctx
    labels = orbital_labels(model)
    projectors, cache = [], {}
    for kpt in basis.kpoints:
        key = id(kpt.mapping)
        if key not in cache:
            Gpk = basis.Gplusk_vectors(kpt)
            Gpk_cart = basis.Gplusk_vectors_cart(kpt)
            gpk_t = Gpk.T.contiguous()
            phi = torch.empty((len(labels), kpt.n_G), dtype=torch.complex128, device=Gpk.device)
            offsets = np.cumsum([0] + [a.psp.count_n_pswfc() for a in model.atoms])
            for group in model.atom_groups:
                psp = model.atoms[group[0]].psp
                ff = (torch.stack(_orbital_rows(psp, Gpk_cart)) / math.sqrt(model.unit_cell_volume)).contiguous()
                nr = ff.shape[0]
                pos = np.ascontiguousarray(np.array([model.positions[ia] for ia in group], dtype=np.float64))
                tmp = torch.empty((nr * len(group), kpt.n_G), dtype=torch.complex128, device=Gpk.device)
                check(ctx.L.dftk_b200_build_projectors(ctx.h, kpt.n_G, _ptr(gpk_t), len(group), _ptr(pos), nr, _ptr(ff),
                                                       _ptr(tmp)), ctx.h)
                for j, ia in enumerate(group):            # the table is atom-major in model order
                    phi[offsets[ia]:offsets[ia] + nr] = tmp[j * nr:(j + 1) * nr]
            cache[key] = ortho_lowdin(ctx, phi)
        projectors.append(cache[key])
    return projectors, labels


def atomic_orbital_projections(basis, psi):
    """dos.jl:198-216: |<φ_j|ψ_n>|² per k-point, (n_bands, n_orb) host arrays, with the labels."""
    projectors, labels = atomic_orbital_projectors(basis)
    out = []
    for phi, p in zip(projectors, psi):
        a = torch.empty((p.shape[0], phi.shape[0]), dtype=torch.complex128, device=phi.device)
        basis.architecture.ctx.zgemm("C", phi, p.contiguous(), a)       # a[n, j] = <φ_j|ψ_n>
        out.append((a.abs() ** 2).cpu().numpy())
    return out, labels


# ------------------------------------------------------------------ symmetry
def wigner_d_matrix(l, Wcart):
    """spherical_harmonics.jl:76-103: D with Y_lm1(W r) = Σ_m2 D[m1, m2] Y_lm2(r) for the real harmonics of
    solid_harmonic_real, by least squares over fixed random unit vectors (exact up to rounding)."""
    if l == 0:
        return np.ones((1, 1))
    # directions over the whole sphere, twice as many as unknowns per row: well conditioned up to l = 3 (positive-octant
    # samples, as in the reference, reach κ(A) > 100 at l = 3); the solve is exact whatever the points
    rng = np.random.default_rng(1234)
    neq = 2 * (2 * l + 1)
    r = rng.standard_normal((neq, 3))
    r /= np.linalg.norm(r, axis=1)[:, None]
    r0 = r @ np.asarray(Wcart, dtype=float).T
    ylm = lambda v: np.stack([solid_harmonic_real(l, m, torch.from_numpy(v)).numpy() for m in range(-l, l + 1)])
    A, B = ylm(r), ylm(r0)                                   # (2l+1, neq)
    if not np.linalg.cond(A) < 100.0:
        raise AssertionError(f"The Wigner matrix computation is badly conditioned. κ(A)={np.linalg.cond(A)}")
    return np.linalg.lstsq(A.T, B.T, rcond=None)[0].T       # B / A


def _symmetry_preimage(positions, position, op, tol=SYMMETRY_TOLERANCE):
    """symmetry.jl:379-396."""
    other = np.linalg.solve(op.W.astype(float), position - op.w)
    dev = [np.max(np.abs((p - other) - np.round(p - other))) for p in positions]
    i = int(np.argmin(dev))
    if dev[i] >= tol:
        raise ValueError("Could not find the preimage of an atom under a symmetry operation")
    return i


def symmetrize_hubbard_n(model, manifold, n, symmetries):
    """symmetry.jl:428-451: n (n_spin, n_atoms, n_atoms, 2l+1, 2l+1); only the on-site blocks are kept (averaged over
    the symmetries as W_D' n_{σ, S⁻¹I} W_D), the inter-site blocks come out zero."""
    positions = [model.positions[ia] for ia in manifold.iatoms]
    out = np.zeros_like(n)
    for op in symmetries:
        Wcart = model.lattice @ op.W @ model.inv_lattice
        D = wigner_d_matrix(manifold.l, Wcart)
        for ia in range(len(positions)):
            ja = _symmetry_preimage(positions, positions[ia], op)
            out[:, ia, ia] += D.T @ n[:, ja, ja] @ D
    return out / len(symmetries)


# ------------------------------------------------------------------ the term
class TermHubbard:
    """hubbard.jl:135-184.  P_vec[ik]: the manifold orbitals of every manifold concatenated, (n_orb, n_pw) device."""

    def __init__(self, basis, hubbard):
        model = basis.model
        self.manifolds = [resolve_hubbard_manifold(m, model) for m in hubbard.manifolds]
        self.U = list(hubbard.U)
        projs, labels = atomic_orbital_projectors(basis)
        self.labels, cols = [], []
        for m in self.manifolds:
            idx = [j for j, lb in enumerate(labels) if lb["iatom"] in m.iatoms and lb["l"] == m.l and lb["n"] == m.i]
            if not idx:
                raise ValueError(f"Projector for manifold (atoms {m.iatoms}, l = {m.l}, i = {m.i}) not found.")
            # atom blocks of 2l+1 columns in manifold.iatoms order (reshape_hubbard_proj)
            order = []
            for ia in m.iatoms:
                order += [j for j in idx if labels[j]["iatom"] == ia]
            self.labels.append([labels[j] for j in order])
            cols += order
        self.columns = cols
        sel = torch.as_tensor(cols, device=basis.architecture.device)
        self.P_vec = [p.index_select(0, sel).contiguous() for p in projs]
        self.n_orb = len(cols)
        self.offsets = np.cumsum([0] + [(2 * m.l + 1) * len(m.iatoms) for m in self.manifolds])

    def coefficients(self, basis, hubbard_n):
        """D[σ] (n_orb × n_orb, block diagonal over manifold atoms, blocks U/2 (I - 2 n_σII)) and the energy."""
        n_spin = basis.model.n_spin_components
        D = np.zeros((n_spin, self.n_orb, self.n_orb), dtype=np.complex128)
        E = 0.0
        filled = basis.model.filled_occupation
        for im, m in enumerate(self.manifolds):
            d = 2 * m.l + 1
            nm = np.asarray(hubbard_n[im])
            for s in range(n_spin):
                for ia in range(len(m.iatoms)):
                    o = self.offsets[im] + ia * d
                    nII = nm[s, ia, ia]
                    D[s, o:o + d, o:o + d] = self.U[im] / 2 * (np.eye(d) - 2 * nII)
                    E += filled * self.U[im] / 2 * float(np.real(np.trace(nII @ (np.eye(d) - nII))))
        return D, E

    def ene_ops(self, basis, psi, occupation, hubbard_n=None, **kw):
        from .terms import NoopOperator, NonlocalOperator
        if hubbard_n is None or not self.U:
            return 0.0, [NoopOperator(basis, k) for k in basis.kpoints]
        D, E = self.coefficients(basis, hubbard_n)
        return E, [NonlocalOperator(basis, k, self.P_vec[ik], D[k.spin], hubbard=True) for ik, k in enumerate(basis.kpoints)]

    def local_occupation(self, basis, psi, occupation):
        """This rank's partial Σ_k w_k Φ'ψ diag(f/filled) ψ'Φ, (n_spin, n_orb, n_orb) complex host array (before the
        sum over ranks)."""
        from .device import orbital_occupation_multi
        filled = basis.model.filled_occupation
        weights = [basis.kweights[ik] * np.asarray(occupation[ik], dtype=float)[:psi[ik].shape[0]] / filled
                   for ik in range(len(basis.kblocks))]
        return orbital_occupation_multi(basis.kblocks, [p.contiguous() for p in psi], weights,
                                        basis.model.n_spin_components, self.n_orb)

    def split(self, basis, n_full):
        """Per manifold (n_spin, n_atoms, n_atoms, 2l+1, 2l+1) views of the summed occupation, symmetrised."""
        out = []
        for im, m in enumerate(self.manifolds):
            d, na = 2 * m.l + 1, len(m.iatoms)
            o = self.offsets[im]
            blk = n_full[:, o:o + na * d, o:o + na * d].reshape(n_full.shape[0], na, d, na, d).transpose(0, 1, 3, 2, 4)
            out.append(symmetrize_hubbard_n(basis.model, m, np.ascontiguousarray(blk), basis.symmetries))
        return out


def compute_hubbard_n(term, basis, psi, occupation):
    """hubbard.jl:201-232: one (n_spin, n_atoms, n_atoms, 2l+1, 2l+1) complex array per manifold.  When (psi, occupation)
    are the ones next_density produced, the sum over ranks already travelled with that step's packed allreduce."""
    c = getattr(basis, "_hubbard_cache", None)
    if c is not None and c["psi"] is psi and c["occupation"] is occupation:
        n_full = c["n"]
    else:
        n_full = term.local_occupation(basis, psi, occupation)
        if basis.comm_kpts.nranks > 1:
            flat = np.concatenate([n_full.real.ravel(), n_full.imag.ravel()])
            flat = np.asarray(basis.comm_kpts.allreduce(flat, "sum"))
            n_full = (flat[:n_full.size] + 1j * flat[n_full.size:]).reshape(n_full.shape)
    return term.split(basis, n_full)
