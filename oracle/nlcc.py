"""Non-linear core correction and the pseudo-atomic valence guess (oracle; test infrastructure only).

Follows src/terms/xc.jl:30-100,206-260 (ρcore in the xc energy, potential and forces) and src/density_methods.jl
(ValenceDensityAuto, CoreDensity) of the reference.  Models without a core density or a pseudo-atomic valence density
give exactly the results of oracle.terms / oracle.forces / oracle.scf, which this module builds on.
"""
import math
import numpy as np
from . import terms as oterms
from . import forces as oforces
from . import scf as oscf


def has(psp, what):
    return bool(getattr(psp, f"has_{what}_density", False))


def core_density(basis):
    """ρcore (n_spin, N): Σ_atoms e^{-2πi G·r} ρ̂core(|G|)/√Ω, split equally over the spins, not renormalised; None
    without core densities."""
    model = basis.model
    if not any(has(a.psp, "core") for a in model.atoms):
        return None
    pn = np.sqrt(np.sum(basis.G_cart ** 2, axis=1))
    rho = np.zeros(basis.N, dtype=complex)
    for ia, atom in enumerate(model.atoms):
        if has(atom.psp, "core"):
            rho += (oterms.structure_factor_cube(basis, model.positions[ia]) * atom.psp.eval_core_density_fourier(pn)
                    / math.sqrt(model.unit_cell_volume))
    rtot = basis.irfft_cube(basis.enforce_real(rho))
    n_spin = model.n_spin_components
    return np.stack([rtot / n_spin] * n_spin)


def xc_potential(basis, rho, rhocore):
    """The xc energy and potential evaluated at ρ + ρcore (gradients included)."""
    return oterms.xc_potential(basis, rho if rhocore is None else rho + rhocore)


def guess_density(basis, magnetic_moments=None):
    """ValenceDensityAuto: the pseudo-atomic valence density where the pseudopotential has one, else the Gaussian."""
    model = basis.model
    if not any(has(a.psp, "valence") for a in model.atoms):
        return oterms.guess_density(basis, magnetic_moments)
    pn = np.sqrt(np.sum(basis.G_cart ** 2, axis=1))

    def superposition(coeffs):
        rho = np.zeros(basis.N, dtype=complex)
        for ia, atom in enumerate(model.atoms):
            if has(atom.psp, "valence"):
                ff = atom.psp.eval_valence_density_fourier(pn)
            else:
                ff = atom.charge_ionic * np.exp(-(pn * oterms.atom_decay_length(atom.n_elec_core, atom.n_elec_valence)) ** 2)
            rho += oterms.structure_factor_cube(basis, model.positions[ia]) * ff * (coeffs[ia] / math.sqrt(model.unit_cell_volume))
        return basis.irfft_cube(basis.enforce_real(rho))

    rtot = superposition(np.ones(len(model.atoms)))
    if model.n_spin_components == 1:
        rho = rtot[None, :]
    else:
        mm = magnetic_moments if magnetic_moments is not None else model.magnetic_moments
        coeffs = [m / a.n_elec_valence for m, a in zip(mm, model.atoms)]
        rspin = superposition(coeffs) if any(c != 0 for c in coeffs) else np.zeros(basis.N)
        rho = np.stack([(rtot + rspin) / 2, (rtot - rspin) / 2])
    Nel = rho.sum() * basis.dvol
    return rho * (model.n_electrons / Nel) if Nel > 0 else rho


def energy_hamiltonian(basis, terms, psi, occupation, rho, eigenvalues=None, eF=None, only_energy=False, rhocore=None):
    """oracle.terms.energy_hamiltonian with the Xc term evaluated at ρ + ρcore."""
    E, blocks = oterms.energy_hamiltonian(basis, terms, psi, occupation, rho, eigenvalues, eF, only_energy)
    if rhocore is None or "Xc" not in basis.model.terms:
        return E, blocks
    _, v0 = oterms.xc_potential(basis, rho)
    E["Xc"], v1 = xc_potential(basis, rho, rhocore)
    E["total"] = sum(v for k, v in E.items() if k != "total")
    if blocks is not None:
        blocks = [oterms.HamiltonianBlock(basis, b.ik, b.kin, b.Vtot - v0[b.kpt.spin] + v1[b.kpt.spin], b.PD)
                  for b in blocks]
    return E, blocks


def self_consistent_field(basis, rho=None, tol=1e-6, maxiter=100, damping=0.8, mixing="simple", rng=None):
    """oracle.scf.self_consistent_field (self_consistent_field.jl:80-289) with ρcore in the Xc term and the
    ValenceDensityAuto guess."""
    model = basis.model
    terms = oterms.Terms(basis)
    rhocore = core_density(basis) if "Xc" in model.terms else None
    rng = rng or np.random.default_rng(7)
    nbandsalg = oscf.AdaptiveBands(model)
    rho = guess_density(basis) if rho is None else rho
    info = dict(psi=None, occupation=None, eigenvalues=None, eF=None, n_iter=0, history_drho=[], converged=False)
    acc = oscf.Anderson(m=10)
    diagtol_max = 0.005

    def fixpoint_map(rho_in):
        if info["n_iter"] <= 1:
            dt = 5 * diagtol_max
        else:
            dt = min(max(min(info["history_drho"]) * 0.2, 100 * np.finfo(float).eps), diagtol_max)
        info["n_iter"] += 1
        _E, blocks = energy_hamiltonian(basis, terms, info["psi"], info["occupation"], rho_in, info["eigenvalues"],
                                        info["eF"], rhocore=rhocore)
        nconv, ncomp = nbandsalg.determine(info["occupation"], info["eigenvalues"], info["psi"])
        if info["psi"] is not None:
            ncomp = max(ncomp, max(p.shape[1] for p in info["psi"]))
        eig = oscf.diagonalize_all_kblocks(blocks, ncomp, psiguess=info["psi"], tol=dt, miniter=1, n_conv_check=nconv,
                                           rng=rng)
        occ, eF = oscf.compute_occupation(basis, eig["λ"], tol_n_elec=nbandsalg.occupation_threshold)
        rho_out = oscf.compute_density(basis, eig["X"], occ, nbandsalg.occupation_threshold)
        info.update(psi=eig["X"], eigenvalues=eig["λ"], occupation=occ, eF=eF, rho_out=rho_out)
        drho = rho_out - rho_in
        info["history_drho"].append(float(np.linalg.norm(drho) * math.sqrt(basis.dvol)))
        mixed = {"simple": lambda: drho, "kerker": lambda: oscf.kerker_mix(basis, drho),
                 "ldos": lambda: oscf.ldos_mix(basis, drho, terms, info)}[mixing]()
        info["converged"] = info["history_drho"][-1] < tol
        return rho_in + mixed

    x = rho
    for _ in range(maxiter):
        fx = fixpoint_map(x)
        if info["converged"]:
            break
        x = acc(x, damping, fx - x)
    E, blocks = energy_hamiltonian(basis, terms, info["psi"], info["occupation"], info["rho_out"], info["eigenvalues"],
                                   info["eF"], rhocore=rhocore)
    return dict(energies=E, ham=blocks, rho=info["rho_out"], psi=info["psi"], eigenvalues=info["eigenvalues"],
                occupation=info["occupation"], eF=info["eF"], converged=info["converged"], n_iter=info["n_iter"],
                terms=terms, rhocore=rhocore, basis=basis)


def forces_xc(basis, rho, rhocore):
    """xc.jl:206-260: F_a,α = -Re Σ_G -2πi G_α e^{-2πi G·r_a} conj(V̄xc(G)) ρ̂core(|G|)/√Ω, V̄xc the spin average of the
    xc potential at ρ + ρcore."""
    model = basis.model
    _, vxc = xc_potential(basis, rho, rhocore)
    v_f = basis.fft_cube(vxc.mean(axis=0))
    pn = np.sqrt(np.sum(basis.G_cart ** 2, axis=1))
    G = basis.G_all.astype(float)
    F = [np.zeros(3) for _ in model.positions]
    for ia, atom in enumerate(model.atoms):
        if has(atom.psp, "core"):
            work = np.exp(-2j * math.pi * (G @ model.positions[ia])) * np.conj(v_f) * atom.psp.eval_core_density_fourier(pn)
            for a in range(3):
                F[ia][a] += -np.real(np.sum(-2j * math.pi * G[:, a] * work) / math.sqrt(model.unit_cell_volume))
    return F


def compute_forces(basis, psi, occupation, rho):
    """oracle.forces.compute_forces plus the Xc (NLCC) term when the model has a core density."""
    total, parts = oforces.compute_forces(basis, psi, occupation, rho)
    rhocore = core_density(basis) if "Xc" in basis.model.terms else None
    if rhocore is not None:
        parts["Xc"] = forces_xc(basis, rho, rhocore)
        total = [t + f for t, f in zip(total, parts["Xc"])]
    return total, parts
