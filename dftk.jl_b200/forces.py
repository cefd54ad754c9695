"""Hellmann-Feynman forces (host-side mirror of src/postprocess/forces.jl:24-58 and the per-term `compute_forces`
methods: local.jl:147-181, nonlocal.jl:49-100, ewald.jl:31,64-168; symmetrize_forces symmetry.jl:379-423).

The two terms that touch grid-sized or orbital-sized data run in libdftk_b200:
  * local:    one kernel pass over the cube per atom (dftk_b200_local_forces),
  * nonlocal: four tensor-core projections P†[ψ, p_x ψ, p_y ψ, p_z ψ] per k-block give the forces on every atom at once
              (dftk_b200_nonlocal_force_rows) instead of the reference's 3·n_atoms full-height GEMM pairs.
Ewald forces are O(n_atoms²) host arithmetic.  Xc contributes only through a model core density (non-linear core
correction of a UPF pseudopotential, xc.jl:206-260); its contraction is that of the local term and uses the same kernel.
Kinetic, Hartree, PspCorrection and Entropy do not contribute.  Forces are in reduced coordinates like the reference;
`compute_forces_cart` converts.
"""
import math
import numpy as np
import torch
from scipy.special import erfc

from ._lib import check
from .device import _ptr
from .basis import estimate_integer_lattice_bounds
from .model import SYMMETRY_TOLERANCE


def forces_local(basis, rho):
    model = basis.model
    ctx = basis.architecture.ctx
    rho_f = basis.fft(rho.sum(dim=0)).reshape(-1)
    pn = basis.G_vectors_cart.norm(dim=1)
    F = [np.zeros(3) for _ in model.positions]
    for group in model.atom_groups:
        ff = model.atoms[group[0]].psp.eval_psp_local_fourier(pn)
        w = (torch.conj(rho_f) * ff / math.sqrt(model.unit_cell_volume)).contiguous()
        pos = np.ascontiguousarray(np.array([model.positions[i] for i in group], dtype=np.float64))
        out = np.zeros((len(group), 3))
        check(ctx.L.dftk_b200_local_forces(basis.fft_grid.h, _ptr(w), len(group), _ptr(pos), _ptr(out)), ctx.h)
        for j, ia in enumerate(group):
            F[ia] = F[ia] + out[j]
    return F


def forces_xc(basis, rho):
    """compute_forces(::TermXc), xc.jl:206-260: the force of the non-linear core correction,
    F_a,α = -Re Σ_G -2πi G_α e^{-2πi G·r_a} conj(V̄xc(G)) ρ̂core(|G|) / sqrt(Ω) with V̄xc the spin average of the xc potential
    at ρ + ρcore -- the contraction of the local-potential force, so it runs through the same kernel.  None without ρcore."""
    model = basis.model
    term = basis.term("Xc")
    if term is None or term.rho_core is None:
        return None
    ctx = basis.architecture.ctx
    _, pot = term.potential(basis, rho)
    v_f = basis.fft(pot.mean(dim=0)).reshape(-1)
    pn = basis.G_vectors_cart.norm(dim=1)
    F = [np.zeros(3) for _ in model.positions]
    for group in model.atom_groups:
        psp = model.atoms[group[0]].psp
        if not getattr(psp, "has_core_density", False):
            continue
        w = (torch.conj(v_f) * psp.eval_psp_core_density_fourier(pn) / math.sqrt(model.unit_cell_volume)).contiguous()
        pos = np.ascontiguousarray(np.array([model.positions[i] for i in group], dtype=np.float64))
        out = np.zeros((len(group), 3))
        check(ctx.L.dftk_b200_local_forces(basis.fft_grid.h, _ptr(w), len(group), _ptr(pos), _ptr(out)), ctx.h)
        for j, ia in enumerate(group):
            F[ia] = F[ia] + out[j]
    return F


def forces_nonlocal(basis, psi, occupation):
    model = basis.model
    ctx = basis.architecture.ctx
    if not any(model.atoms[g[0]].psp.count_n_proj() for g in model.atom_groups):
        return None
    # projector rows are ordered (group, atom in group, l, m, i) like TermAtomicNonlocal builds P
    owners = []
    for group in model.atom_groups:
        n = model.atoms[group[0]].psp.count_n_proj()
        for ia in group:
            owners += [ia] * n
    owners = np.array(owners, dtype=np.int64)
    F = np.zeros((len(model.positions), 3))
    for ik, kb in enumerate(basis.kblocks):
        if kb.n_proj == 0:
            continue
        assert kb.n_proj == len(owners)
        occ = np.asarray(occupation[ik], dtype=np.float64)
        nb = int(np.max(np.nonzero(occ)[0]) + 1) if np.any(occ != 0) else 0
        if nb == 0:
            continue
        w = np.ascontiguousarray(occ[:nb] * basis.kweights[ik])
        gpk = basis.Gplusk_vectors(basis.kpoints[ik]).T.contiguous()            # (3, n_pw) reduced G+k
        rows = np.zeros((3, kb.n_proj))
        check(ctx.L.dftk_b200_nonlocal_force_rows(kb.h, _ptr(psi[ik][:nb].contiguous()), _ptr(w), nb, _ptr(gpk),
                                                  _ptr(rows)), ctx.h)
        for a in range(3):
            F[:, a] += np.bincount(owners, weights=rows[a], minlength=F.shape[0])
    F = np.asarray(basis.comm_kpts.sum(F))                                    # mpi_sum!(forces, comm_kpts)
    return symmetrize_forces(basis, [F[i] for i in range(F.shape[0])])


def ewald_parameters(lattice, positions, eta=None):
    """η and the summation limits of ewald.jl:86-104."""
    lattice = np.asarray(lattice, dtype=float)
    pos = np.array([np.asarray(p, dtype=float) for p in positions])
    recip = 2 * math.pi * np.linalg.inv(lattice.T)
    if eta is None:
        eta = math.sqrt(math.sqrt(1.69 * np.linalg.norm(recip / (2 * math.pi)) / np.linalg.norm(lattice))) / 2
    max_exp = -math.log(np.finfo(float).eps) + 5
    Glims = estimate_integer_lattice_bounds(recip, math.sqrt(max_exp) * 2 * eta)
    poslims = [float(np.max(pos[:, i][:, None] - pos[:, i][None, :])) for i in range(3)]
    Rlims = estimate_integer_lattice_bounds(lattice, math.sqrt(max_exp) / eta, poslims)
    return eta, Glims, Rlims


def energy_forces_ewald_device(ctx, lattice, charges, positions, eta=None):
    """energy_forces_ewald (ewald.jl:64-168, q = 0) on the device: the O(n_atoms² n_R) real-space sum and the O(n_atoms n_G)
    reciprocal sum are one kernel each (dftk_b200_ewald); η and the limits are the host's."""
    eta, Glims, Rlims = ewald_parameters(lattice, positions, eta)
    n = len(positions)
    lat = np.asfortranarray(np.asarray(lattice, dtype=np.float64))
    ch = np.ascontiguousarray(charges, dtype=np.float64)
    pos = np.ascontiguousarray(np.array([np.asarray(p, dtype=np.float64) for p in positions]))
    gl, rl = np.array(Glims, dtype=np.int32), np.array(Rlims, dtype=np.int32)
    e, f = np.zeros(1), np.zeros((n, 3))
    check(ctx.L.dftk_b200_ewald(ctx.h, _ptr(lat), n, _ptr(ch), _ptr(pos), float(eta), _ptr(gl), _ptr(rl), _ptr(e), _ptr(f)), ctx.h)
    return float(e[0]), [f[i].copy() for i in range(n)]


def energy_forces_ewald(lattice, charges, positions, eta=None):
    """ewald.jl:64-168 for q = 0 (energy as terms.energy_ewald, plus the forces): vectorised NumPy on the host -- the form the
    CPU-only unit tests compare with the oracle; the product's terms use `energy_forces_ewald_device`."""
    lattice = np.asarray(lattice, dtype=float)
    charges = np.asarray(charges, dtype=float)
    pos = np.array([np.asarray(p, dtype=float) for p in positions])
    n = len(pos)
    recip = 2 * math.pi * np.linalg.inv(lattice.T)
    if eta is None:
        eta = math.sqrt(math.sqrt(1.69 * np.linalg.norm(recip / (2 * math.pi)) / np.linalg.norm(lattice))) / 2
    max_exp = -math.log(np.finfo(float).eps) + 5
    Glims = estimate_integer_lattice_bounds(recip, math.sqrt(max_exp) * 2 * eta)
    poslims = [float(np.max(pos[:, i][:, None] - pos[:, i][None, :])) for i in range(3)]
    Rlims = estimate_integer_lattice_bounds(lattice, math.sqrt(max_exp) / eta, poslims)
    vol = abs(np.linalg.det(lattice))
    G = np.stack(np.meshgrid(*[np.arange(-g, g + 1) for g in Glims], indexing="ij"), -1).reshape(-1, 3)
    G = G[np.any(G != 0, axis=1)].astype(float)
    Gsq = np.sum((G @ recip.T) ** 2, axis=1)
    damp = np.exp(-Gsq / (4 * eta ** 2)) / Gsq
    cs, sn = np.zeros(len(G)), np.zeros(len(G))
    for c in range(0, n, 32):
        ph = 2 * math.pi * (G @ pos[c:c + 32].T)
        cs += (np.cos(ph) * charges[c:c + 32]).sum(axis=1)
        sn += (np.sin(ph) * charges[c:c + 32]).sum(axis=1)
    sum_recip = -(charges.sum() ** 2 / (4 * eta ** 2)) + np.sum((cs ** 2 + sn ** 2) * damp)
    F_recip = np.zeros((n, 3))
    for c in range(0, n, 32):
        ph = 2 * math.pi * (G @ pos[c:c + 32].T)
        coeff = charges[c:c + 32] * 2 * math.pi * (-cs[:, None] * np.sin(ph) + sn[:, None] * np.cos(ph)) * damp[:, None]
        F_recip[c:c + 32] = -(coeff.T @ G)
    sum_recip *= 4 * math.pi / vol
    F_recip *= 4 * math.pi / vol
    sum_real = -2 * eta / math.sqrt(math.pi) * np.sum(charges ** 2)
    F_real = np.zeros((n, 3))
    R = np.stack(np.meshgrid(*[np.arange(-g, g + 1) for g in Rlims], indexing="ij"), -1).reshape(-1, 3).astype(float)
    Rcart = R @ lattice.T
    nonzero = np.any(R != 0, axis=1)
    for i in range(n):
        d = ((pos[i] - pos) @ lattice.T)[:, None, :] - Rcart[None, :, :]     # Δr (n_atoms, n_R, 3)
        dist = np.linalg.norm(d, axis=2)
        mask = np.ones_like(dist, dtype=bool)
        mask[i, ~nonzero] = False
        dist = np.where(mask, dist, 1.0)
        zz = charges[i] * charges[:, None]
        e = np.where(mask, zz * erfc(eta * dist) / dist, 0.0)
        sum_real += np.sum(e)
        dE = np.where(mask, (zz * eta * (-2 * np.exp(-(eta * dist) ** 2) / math.sqrt(math.pi)) - e) / dist, 0.0)
        F_real[i] = -(lattice.T @ np.einsum("jr,jrc->c", dE / dist, d))
    return (sum_recip + sum_real) / 2, [F_recip[i] + F_real[i] for i in range(n)]


def find_symmetry_preimage(positions_group, position, symop, tol_symmetry=SYMMETRY_TOLERANCE):
    other = np.linalg.solve(symop.W.astype(float), position - symop.w)
    dev = [float(np.max(np.abs((at - other) - np.round(at - other)))) for at in positions_group]
    i = int(np.argmin(dev))
    assert dev[i] < 10 * tol_symmetry
    return i


def symmetrize_forces(basis_or_model, forces, symmetries=None):
    """symmetry.jl:399-423: F_sym[a] = 1/n_sym Σ_s W_s^{-T} F[preimage_s(a)] in reduced coordinates."""
    model = getattr(basis_or_model, "model", basis_or_model)
    if symmetries is None:
        symmetries = basis_or_model.symmetries
    out = [np.zeros(3) for _ in forces]
    for group in model.atom_groups:
        pg = [model.positions[i] for i in group]
        for s in symmetries:
            WinvT = np.linalg.inv(s.W.astype(float).T)
            for idx, p in enumerate(pg):
                j = find_symmetry_preimage(pg, p, s)
                out[group[idx]] = out[group[idx]] + WinvT @ forces[group[j]]
    return [f / len(symmetries) for f in out]


def compute_forces(basis_or_scfres, psi=None, occupation=None, *, rho=None, per_term=False):
    """compute_forces(basis, ψ, occupation; ρ) / compute_forces(scfres) -- reduced coordinates."""
    if isinstance(basis_or_scfres, dict):
        res = basis_or_scfres
        basis, psi, occupation, rho = res["basis"], res["psi"], res["occupation"], res["rho"]
    else:
        basis = basis_or_scfres
    model = basis.model
    if "Hubbard" in model.term_names:
        # the ortho-atomic orbitals depend on every position through S^{-1/2}: no Hubbard force is implemented, and
        # leaving the term out would return forces of a different energy
        raise NotImplementedError("compute_forces: forces of a model with a Hubbard term are not implemented")
    parts = {}
    for name in model.term_types:
        if name == "AtomicLocal":
            parts[name] = forces_local(basis, rho)
        elif name == "AtomicNonlocal":
            f = forces_nonlocal(basis, psi, occupation)
            if f is not None:
                parts[name] = f
        elif name == "Ewald":
            parts[name] = energy_forces_ewald_device(basis.architecture.ctx, model.lattice, [a.charge_ionic() for a in model.atoms],
                                                     model.positions)[1]
        elif name == "Xc":
            f = forces_xc(basis, rho)
            if f is not None:
                parts[name] = f
    total = [sum((p[i] for p in parts.values()), np.zeros(3)) for i in range(len(model.positions))]
    return (total, parts) if per_term else total


def compute_forces_cart(basis_or_scfres, psi=None, occupation=None, *, rho=None):
    """covector_red_to_cart: F_cart = inv(lattice)' F_red (Hartree / bohr)."""
    basis = basis_or_scfres["basis"] if isinstance(basis_or_scfres, dict) else basis_or_scfres
    inv_lat_T = basis.model.inv_lattice.T
    return [inv_lat_T @ f for f in compute_forces(basis_or_scfres, psi, occupation, rho=rho)]
