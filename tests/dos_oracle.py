"""Oracle for the densities of states (test infrastructure only): a literal NumPy restatement of src/postprocess/dos.jl,
loop for loop, that never imports the product.  The smearing derivatives come from smearing_oracle.  Inputs are plain
data: per k-block of the basis its spin, k-point weight and eigenvalues; for the LDOS the band densities |ψ_kn(r)|²/Ω,
for the PDOS the projections |<φ_p|ψ_kn>|²."""
import numpy as np

import smearing_oracle as so


def _check(smearing, temperature, what):
    if temperature == 0 or smearing == "None":
        raise ValueError(f"{what} only supports finite temperature")


def ldos_weight(εnk, ε, filled, smearing, temperature):
    """dos.jl compute_ldos: -filled / T f'((εnk - ε) / T)."""
    return -filled / temperature * float(so.occupation_derivative(smearing, np.array((εnk - ε) / temperature)))


def compute_dos(ε, spins, kweights, eigenvalues, n_spin, filled, smearing, temperature):
    """dos.jl compute_dos at one energy: (n_spin,)."""
    _check(smearing, temperature, "compute_dos")
    D = np.zeros(n_spin)
    for σ, wk, εk in zip(spins, kweights, eigenvalues):
        for εnk in εk:
            D[σ] -= filled * wk / temperature * float(so.occupation_derivative(smearing, np.array((εnk - ε) / temperature)))
    return D


def compute_ldos_unsymmetrised(ε, spins, kweights, eigenvalues, band_densities, n_spin, filled, smearing, temperature,
                               weight_threshold=np.finfo(float).eps):
    """dos.jl compute_ldos before the symmetrisation of compute_density: band_densities[ik] (n_bands, N)."""
    _check(smearing, temperature, "compute_ldos")
    N = band_densities[0].shape[1]
    rho = np.zeros((n_spin, N))
    for σ, wk, εk, dk in zip(spins, kweights, eigenvalues, band_densities):
        for n, εnk in enumerate(εk[:dk.shape[0]]):
            w = ldos_weight(εnk, ε, filled, smearing, temperature)
            if abs(w) >= weight_threshold:
                rho[σ] += w * wk * dk[n]
    return rho


def compute_pdos(εs, spins, kweights, eigenvalues, projections, n_spin, filled, smearing, temperature):
    """dos.jl compute_pdos: projections[ik] (n_bands, n_orb) -> (n_ε, n_orb, n_spin)."""
    _check(smearing, temperature, "compute_pdos")
    n_orb = projections[0].shape[1]
    D = np.zeros((len(εs), n_orb, n_spin))
    for iε, ε in enumerate(εs):
        for σ, wk, εk, pk in zip(spins, kweights, eigenvalues, projections):
            for n, εnk in enumerate(εk[:pk.shape[0]]):
                enred = (εnk - ε) / temperature
                for p in range(pk.shape[1]):
                    D[iε, p, σ] -= (filled * wk * pk[n, p] / temperature
                                    * float(so.occupation_derivative(smearing, np.array(enred))))
    return D


def sum_pdos(pdos, labels, n_ε, filters):
    """dos.jl sum_pdos."""
    out = np.zeros((n_ε, pdos.shape[2]))
    for σ in range(pdos.shape[2]):
        for j, orb in enumerate(labels):
            if any(f(orb) for f in filters):
                out[:, σ] += pdos[:, j, σ]
    return out
