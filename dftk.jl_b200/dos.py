"""Densities of states (mirror of src/postprocess/dos.jl): compute_dos, compute_ldos, compute_pdos and sum_pdos.

All three share the weight of band n of k-point k at energy ε_j,
    W[j, kn] = -filled / T · f'((ε_kn - ε_j) / T),
times the k-point weight: the DOS is Σ_kn of it, the PDOS its product with the projections |<φ_p|ψ_kn>|², both on the host,
and the LDOS its product with the band densities |ψ_kn(r)|².  For many energies the LDOS takes one pass over the bands
(dftk_b200_ldos_accumulate_multi): |ψ_kn(r)|² does not depend on ε, so every band is transformed once and the energies
come from one real FP64 tensor-core product, where a loop of compute_density calls would transform every band per energy.
k-sums go over basis.comm_kpts by one allreduce."""
import collections

import numpy as np
import torch

from .basis import PlaneWaveBasis
from .densities import compute_density, symmetrize_rho
from .terms import occupation_derivative

PdosResult = collections.namedtuple("PdosResult", ["pdos", "projector_labels", "εs"])


def _smearing_and_temperature(basis, smearing, temperature, what):
    smearing = basis.model.smearing if smearing is None else smearing
    temperature = basis.model.temperature if temperature is None else float(temperature)
    if temperature == 0 or smearing == "None":
        raise ValueError(f"{what} only supports finite temperature")
    return smearing, temperature


def dos_weights(basis, eigenvalues, εs, smearing, temperature):
    """-filled/T f'((ε_kn - ε_j)/T) per block of this rank: a list of (n_ε, n_bands_k) arrays, without the k-point weight."""
    filled = basis.model.filled_occupation
    εs = np.asarray(εs, dtype=float).reshape(-1)
    return [-filled / temperature * occupation_derivative(smearing, (np.asarray(e, dtype=float)[None, :] - εs[:, None]) / temperature)
            for e in eigenvalues]


def _spin_sum(basis, per_block, shape):
    """Σ over the blocks of each spin of per_block[i] (arrays of `shape`), over all ranks: (*shape, n_spin)."""
    out = np.zeros(tuple(shape) + (basis.model.n_spin_components,))
    for kpt, x in zip(basis.kpoints, per_block):
        out[..., kpt.spin] += x
    return basis.comm_kpts.allreduce(out)


def compute_dos(ε, basis=None, eigenvalues=None, *, smearing=None, temperature=None):
    """Total density of states at ε (a number or a 1-D array): shape (n_spin,), or (n_ε, n_spin) for an array.
    `compute_dos(scfres[, ε])` (ε defaults to scfres["eF"]) takes basis and eigenvalues from an SCF result."""
    if isinstance(ε, dict):
        scfres = ε
        ε = scfres["eF"] if basis is None else basis
        return compute_dos(ε, scfres["basis"], scfres["eigenvalues"], smearing=smearing, temperature=temperature)
    smearing, temperature = _smearing_and_temperature(basis, smearing, temperature, "compute_dos")
    εs = np.asarray(ε, dtype=float)
    W = dos_weights(basis, eigenvalues, εs, smearing, temperature)
    D = _spin_sum(basis, [wk * w.sum(axis=1) for wk, w in zip(basis.kweights, W)], (εs.size,))
    return D[0] if εs.ndim == 0 else D


def compute_ldos(ε, basis=None, eigenvalues=None, psi=None, *, smearing=None, temperature=None,
                 weight_threshold=np.finfo(float).eps, **kwargs):
    """Local density of states at ε, symmetrised like compute_density.  A number ε gives (n_spin, N) on the device, a 1-D
    array (n_ε, n_spin, N) from one pass over the bands.  Weights below `weight_threshold` are screened away; a band screened
    away at every energy is not transformed.  `compute_ldos(scfres[, ε])` (ε defaults to scfres["eF"]) takes the rest from an SCF result.

    The form `compute_ldos(basis, eF, eigenvalues, psi, *, temperature)` of LdosMixing (Gaussian smearing) is kept."""
    if isinstance(ε, PlaneWaveBasis):
        from .scf import compute_ldos as gaussian_ldos
        return gaussian_ldos(ε, basis, eigenvalues, psi, temperature=temperature, weight_threshold=weight_threshold, **kwargs)
    if kwargs:
        raise TypeError(f"compute_ldos: unexpected arguments {sorted(kwargs)}")
    if isinstance(ε, dict):
        scfres = ε
        ε = scfres["eF"] if basis is None else basis
        return compute_ldos(ε, scfres["basis"], scfres["eigenvalues"], scfres["psi"], smearing=smearing,
                            temperature=temperature, weight_threshold=weight_threshold)
    smearing, temperature = _smearing_and_temperature(basis, smearing, temperature, "compute_ldos")
    εs = np.asarray(ε, dtype=float)
    W = [w[:, :p.shape[0]] for w, p in zip(dos_weights(basis, eigenvalues, εs, smearing, temperature), psi)]
    if εs.ndim == 0:
        return compute_density(basis, psi, [w[0] for w in W], occupation_threshold=weight_threshold)
    if getattr(basis, "comm_slab", None) is not None:
        raise NotImplementedError("compute_ldos at several energies does not support slab-distributed bases")
    from .device import ldos_accumulate_multi
    dev = basis.architecture.device
    n_spin, n_e = basis.model.n_spin_components, εs.size
    ld_w = max([1] + [p.shape[0] for p in psi])
    Wh = np.zeros((n_e, len(basis.kblocks), ld_w))
    for i, (w, wk) in enumerate(zip(W, basis.kweights)):
        Wh[:, i, :w.shape[1]] = np.where(np.abs(w) >= weight_threshold, w * wk, 0.0)
    ldos = torch.zeros((n_e, n_spin, basis.N), dtype=torch.float64, device=dev)
    ldos_accumulate_multi(basis.kblocks, [p.contiguous() for p in psi], torch.from_numpy(Wh).to(dev), ldos)
    if basis.comm_kpts.nranks > 1:
        basis.comm_kpts.n_collectives += 1
        basis.architecture.ctx.allreduce(ldos, "sum")
    for j in range(n_e):
        ldos[j] = symmetrize_rho(basis, ldos[j])
    return ldos


def compute_pdos(εs, basis=None, psi=None, eigenvalues=None, *, positions=None, smearing=None, temperature=None):
    """Projected density of states on the ortho-atomic orbitals of every atom: (pdos[n_ε, n_orb, n_spin],
    projector_labels, εs).  `compute_pdos(scfres[, εs])` (εs defaults to [scfres["eF"]]) takes the rest from an SCF result."""
    if isinstance(εs, dict):
        scfres = εs
        εs = [scfres["eF"]] if basis is None else basis
        return compute_pdos(εs, scfres["basis"], scfres["psi"], scfres["eigenvalues"], positions=positions,
                            smearing=smearing, temperature=temperature)
    if positions is not None and not (len(positions) == len(basis.model.positions) and all(
            np.array_equal(np.asarray(p, dtype=float), q) for p, q in zip(positions, basis.model.positions))):
        raise NotImplementedError("compute_pdos supports only the model's own atomic positions")
    smearing, temperature = _smearing_and_temperature(basis, smearing, temperature, "compute_pdos")
    from .hubbard import atomic_orbital_projections
    εs = np.atleast_1d(np.asarray(εs, dtype=float))
    projections, labels = atomic_orbital_projections(basis, psi)
    W = dos_weights(basis, eigenvalues, εs, smearing, temperature)
    pdos = _spin_sum(basis, [wk * w[:, :pr.shape[0]] @ pr for wk, w, pr in zip(basis.kweights, W, projections)],
                     (εs.size, len(labels)))
    return PdosResult(pdos, labels, εs)


def sum_pdos(pdos_res, projector_filters):
    """Σ of the PDOS columns whose label matches any of the filters (functions of a label): (n_ε, n_spin)."""
    pdos, labels, εs = pdos_res
    out = np.zeros((len(εs), pdos.shape[2]))
    for j, orb in enumerate(labels):
        if any(f(orb) for f in projector_filters):
            out += pdos[:, j, :]
    return out
