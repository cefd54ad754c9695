"""NumPy restatement of DFT+U for the tests: pseudo-atomic orbitals of a UPF file (PspUpf.jl:140-155,218-223),
ortho-atomic projectors (dos.jl:156-196, ortho.jl), occupation matrices, their symmetrisation and the Hubbard energy
and operator (hubbard.jl, symmetry.jl:428-451, spherical_harmonics.jl:76-103).  It works on the oracle's basis objects
and shares no code with the package: the radial transforms go through oracle.psp_upf.hankel (scipy Bessel functions).
Orbital tables are (n_G, n_orb) and orbitals (n_G, n_bands), column = vector, as in the oracle."""
import math
import xml.etree.ElementTree as ET
import numpy as np

from oracle.psp_upf import hankel, psp_quadrature_weights
from oracle.psp_hgh import solid_harmonic_real

SYMMETRY_TOLERANCE = 1e-5


def parse_pswfc(text):
    """[(label, l, occupation, rχ)] of PP_PSWFC in file order."""
    root = ET.fromstring(text)
    wfc = root.find("PP_PSWFC")
    out = []
    for c in (wfc if wfc is not None else []):
        if c.tag.startswith("PP_CHI"):
            out.append((c.get("label").strip(), int(c.get("l")), float(c.get("occupation")),
                        np.array(c.text.split(), dtype=float)))
    return out


class Orbitals:
    """The orbitals of one pseudopotential kept by the reference: l <= lmax, r²χ = r·(rχ), grouped by l."""

    def __init__(self, text, psp):
        self.psp = psp
        r = psp.rgrid
        self.by_l = [[] for _ in range(psp.lmax + 1)]
        for label, l, _occ, rchi in parse_pswfc(text):
            if l <= psp.lmax:
                self.by_l[l].append((label, r * rchi[:len(r)]))

    def fourier(self, i, l, p):
        r2chi = self.by_l[l][i - 1][1]
        r = self.psp.rgrid
        return hankel(r, r2chi, l, p, psp_quadrature_weights(r, len(r)))


def raw_table(basis, kpt, orbitals):
    """Unorthogonalised table and labels; orbitals[ia]: the Orbitals of atom ia."""
    m = basis.model
    Gpk = kpt.G_vectors + kpt.coordinate
    Gc = basis.Gplusk_cart(kpt)
    pn = np.sqrt(np.sum(Gc ** 2, axis=1))
    cols, labels = [], []
    for ia, orb in enumerate(orbitals):
        sf = np.exp(-2j * math.pi * (Gpk @ m.positions[ia])) / math.sqrt(m.unit_cell_volume)
        for l in range(len(orb.by_l)):
            for n in range(1, len(orb.by_l[l]) + 1):
                rad = orb.fourier(n, l, pn)
                for mm in range(-l, l + 1):
                    cols.append(rad * ((-1j) ** l) * solid_harmonic_real(l, mm, Gc) * sf)
                    labels.append((ia, n, l, mm, orb.by_l[l][n - 1][0]))
    return np.stack(cols, axis=1), labels


def ortho_lowdin(phi):
    ev, U = np.linalg.eigh(phi.conj().T @ phi)
    assert np.min(np.abs(ev)) > np.finfo(float).eps * np.max(np.abs(ev))
    return phi @ ((U * ev ** -0.5) @ U.conj().T)


def projectors(basis, orbitals):
    """Per k-point the Löwdin-orthonormalised complete table, and the labels (iatom, n, l, m, label)."""
    out = []
    for kpt in basis.kpoints:
        phi, labels = raw_table(basis, kpt, orbitals)
        out.append(ortho_lowdin(phi))
    return out, labels


class Manifold:
    def __init__(self, iatoms, l, i, U):
        self.iatoms, self.l, self.i, self.U = list(iatoms), l, i, float(U)


def manifold_columns(labels, man):
    cols = []
    for ia in man.iatoms:
        cols += [j for j, lb in enumerate(labels) if lb[0] == ia and lb[2] == man.l and lb[1] == man.i]
    assert len(cols) == len(man.iatoms) * (2 * man.l + 1)
    return cols


def wigner_d_matrix(l, Wcart):
    """The real-harmonic representation D of Wcart, Y(W r) = D Y(r), solved exactly on 2l+1 generic directions."""
    if l == 0:
        return np.ones((1, 1))
    rng = np.random.default_rng(7)
    r = rng.standard_normal((2 * l + 1, 3))
    r /= np.linalg.norm(r, axis=1)[:, None]
    Y = lambda v: np.stack([solid_harmonic_real(l, m, v) for m in range(-l, l + 1)])
    return Y(r @ np.asarray(Wcart).T) @ np.linalg.inv(Y(r))


def symmetrize(model, man, n, symmetries):
    pos = [model.positions[ia] for ia in man.iatoms]
    out = np.zeros_like(n)
    for op in symmetries:
        D = wigner_d_matrix(man.l, model.lattice @ op.W @ np.linalg.inv(model.lattice))
        for ia in range(len(pos)):
            other = np.linalg.solve(op.W.astype(float), pos[ia] - op.w)
            dev = [np.max(np.abs((p - other) - np.round(p - other))) for p in pos]
            ja = int(np.argmin(dev))
            assert dev[ja] < SYMMETRY_TOLERANCE
            out[:, ia, ia] += D.T @ n[:, ja, ja] @ D
    return out / len(symmetries)


def hubbard_n(basis, projs, labels, man, psi, occupation, symmetries=None):
    """(n_spin, n_atoms, n_atoms, 2l+1, 2l+1) of one manifold; psi[ik]: (n_G, n_bands)."""
    m = basis.model
    d, na = 2 * man.l + 1, len(man.iatoms)
    cols = manifold_columns(labels, man)
    n = np.zeros((m.n_spin_components, na, na, d, d), dtype=complex)
    for ik, kpt in enumerate(basis.kpoints):
        a = projs[ik][:, cols].conj().T @ psi[ik]                      # <φ|ψ>
        w = basis.kweights[ik] * np.asarray(occupation[ik])[:psi[ik].shape[1]] / m.filled_occupation
        full = (a * w) @ a.conj().T
        n[kpt.spin] += full.reshape(na, d, na, d).transpose(0, 2, 1, 3)
    return symmetrize(m, man, n, basis.symmetries if symmetries is None else symmetries)


def energy_and_coefficients(basis, manifolds, ns):
    """E_U and, per spin, D over the concatenated manifold columns (blocks U/2 (I - 2 n_σII))."""
    m = basis.model
    sizes = [(2 * man.l + 1) * len(man.iatoms) for man in manifolds]
    D = np.zeros((m.n_spin_components, sum(sizes), sum(sizes)), dtype=complex)
    E, o = 0.0, 0
    for man, n in zip(manifolds, ns):
        d = 2 * man.l + 1
        for s in range(m.n_spin_components):
            for ia in range(len(man.iatoms)):
                nII = n[s, ia, ia]
                D[s, o + ia * d:o + (ia + 1) * d, o + ia * d:o + (ia + 1) * d] = man.U / 2 * (np.eye(d) - 2 * nII)
                E += m.filled_occupation * man.U / 2 * np.real(np.trace(nII @ (np.eye(d) - nII)))
        o += sizes[manifolds.index(man)]
    return E, D


def manifold_table(projs, labels, manifolds):
    cols = sum((manifold_columns(labels, man) for man in manifolds), [])
    return [p[:, cols] for p in projs]


# ------------------------------------------------------------------ SCF (self_consistent_field.jl:19-45,168,200-289)
class HubbardBlock:
    """An oracle Hamiltonian block plus the Hubbard operator Φ D Φ'."""

    def __init__(self, blk, Phi, D):
        self.blk, self.Phi, self.D = blk, Phi, D
        self.kpt, self.kin, self.ik, self.shape = blk.kpt, blk.kin, blk.ik, blk.shape

    def matmul(self, X):
        return self.blk.matmul(X) + self.Phi @ (self.D @ (self.Phi.conj().T @ X))

    __matmul__ = matmul


def scf(basis, orbitals, manifolds, tol=1e-10, maxiter=100, damping=0.8):
    """oracle.nlcc.self_consistent_field with the Hubbard term: the Hamiltonian of a step uses the previous step's
    occupation (none in the first step), which is recomputed from the new orbitals after every density update and never
    mixed; the final energies and Hamiltonian use the last one."""
    from oracle import nlcc, scf as oscf, terms as oterms
    model = basis.model
    terms = oterms.Terms(basis)
    rhocore = nlcc.core_density(basis) if "Xc" in model.terms else None
    projs, labels = projectors(basis, orbitals)
    Phi = manifold_table(projs, labels, manifolds)
    rng = np.random.default_rng(7)
    nbandsalg = oscf.AdaptiveBands(model)
    info = dict(psi=None, occupation=None, eigenvalues=None, eF=None, n_iter=0, history_drho=[], converged=False, n=None)
    acc = oscf.Anderson(m=10)

    def ham(psi, occ, rho, eigenvalues, eF, n, only_energy=False):
        E, blocks = nlcc.energy_hamiltonian(basis, terms, psi, occ, rho, eigenvalues, eF, only_energy=only_energy,
                                            rhocore=rhocore)
        EU, D = (0.0, None) if n is None else energy_and_coefficients(basis, manifolds, n)
        E["Hubbard"] = EU
        E["total"] = sum(v for k, v in E.items() if k != "total")
        if blocks is not None and D is not None:
            blocks = [HubbardBlock(b, Phi[b.ik], D[b.kpt.spin]) for b in blocks]
        return E, blocks

    def fixpoint_map(rho_in):
        dt = 0.025 if info["n_iter"] <= 1 else min(max(min(info["history_drho"]) * 0.2, 100 * np.finfo(float).eps), 0.005)
        info["n_iter"] += 1
        _E, blocks = ham(info["psi"], info["occupation"], rho_in, info["eigenvalues"], info["eF"], info["n"])
        nconv, ncomp = nbandsalg.determine(info["occupation"], info["eigenvalues"], info["psi"])
        if info["psi"] is not None:
            ncomp = max(ncomp, max(p.shape[1] for p in info["psi"]))
        eig = oscf.diagonalize_all_kblocks(blocks, ncomp, psiguess=info["psi"], tol=dt, miniter=1, n_conv_check=nconv,
                                           rng=rng)
        occ, eF = oscf.compute_occupation(basis, eig["λ"], tol_n_elec=nbandsalg.occupation_threshold)
        rho_out = oscf.compute_density(basis, eig["X"], occ, nbandsalg.occupation_threshold)
        n = [hubbard_n(basis, projs, labels, m, eig["X"], occ) for m in manifolds]
        info.update(psi=eig["X"], eigenvalues=eig["λ"], occupation=occ, eF=eF, rho_out=rho_out, n=n)
        drho = rho_out - rho_in
        info["history_drho"].append(float(np.linalg.norm(drho) * math.sqrt(basis.dvol)))
        info["converged"] = info["history_drho"][-1] < tol
        return rho_in + drho

    x = nlcc.guess_density(basis)
    for _ in range(maxiter):
        fx = fixpoint_map(x)
        if info["converged"]:
            break
        x = acc(x, damping, fx - x)
    E, blocks = ham(info["psi"], info["occupation"], info["rho_out"], info["eigenvalues"], info["eF"], info["n"])
    return dict(energies=E, ham=blocks, rho=info["rho_out"], psi=info["psi"], eigenvalues=info["eigenvalues"],
                occupation=info["occupation"], eF=info["eF"], converged=info["converged"], n_iter=info["n_iter"],
                hubbard_n=info["n"], projectors=projs, labels=labels)
