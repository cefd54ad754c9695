"""Hamiltonian / DftHamiltonianBlock / energy_hamiltonian (host-side mirror of
src/terms/Hamiltonian.jl:22-57,137-236).  `mul!(Hψ, H::DftHamiltonianBlock, ψ)` is one C-ABI call
(dftk_b200_apply_h) that runs the batched FFT pipeline + fused kinetic/local scalings + nonlocal GEMMs."""
import math
import numpy as np
import torch

from .terms import (RealSpaceMultiplication, FourierMultiplication, NonlocalOperator, NoopOperator)


class Energies(dict):
    """src/Energies.jl: named energy container with a `.total`."""

    @property
    def total(self):
        return sum(self.values())


class DftHamiltonianBlock:
    def __init__(self, basis, ik, operators, pot_cache=None):
        self.basis, self.ik, self.kpoint = basis, ik, basis.kpoints[ik]
        self.operators = operators
        ops = [o for o in operators if not isinstance(o, NoopOperator)]
        fourier = [o for o in ops if isinstance(o, FourierMultiplication)]
        real = [o for o in ops if isinstance(o, RealSpaceMultiplication)]
        nonloc = [o for o in ops if isinstance(o, NonlocalOperator) and not o.hubbard]
        hub = [o for o in ops if isinstance(o, NonlocalOperator) and o.hubbard]
        if (len(fourier) > 1 or len(nonloc) > 1 or len(hub) > 1
                or len(fourier) + len(real) + len(nonloc) + len(hub) != len(ops)):
            raise NotImplementedError("only DFT Hamiltonians (one Fourier multiplication, local potentials, "
                                      "at most one atomic and one Hubbard nonlocal operator) are supported by this GPU back end")
        self.fourier_op = fourier[0] if fourier else None
        self.nonlocal_op = nonloc[0] if nonloc else None
        self.hubbard_op = hub[0] if hub else None
        # optimize_operators (operators.jl:213-222): sum all real-space multiplications
        self.local_op = None
        if real:
            # all k-blocks of one spin share the same term potentials: sum them once (keyed by the storage they view)
            key = tuple((o.potential.data_ptr(), o.potential.numel()) for o in real)
            pot = pot_cache.get(key) if pot_cache is not None else None
            if pot is None:
                pot = real[0].potential
                for o in real[1:]:
                    pot = pot + o.potential
                pot = pot.contiguous()
                if pot_cache is not None:
                    pot_cache[key] = pot
            self.local_op = RealSpaceMultiplication(basis, self.kpoint, pot)
        self.kblock = basis.kblocks[ik]

    def bind(self):
        """Install this block's local potential on the shared device k-block.  A Hamiltonian is a value in the
        reference: several may be alive at once (scfres.ham, info.ham of a callback, ham(ρ1) vs ham(ρ2)), so the
        potential travels with the block and is (re)installed before every device call; the k-block skips the copy
        when it already holds this very tensor."""
        if self.local_op is None:
            self.kblock.set_potential(None)
        else:
            # all blocks of a spin channel share the summed potential: one device copy per (grid, spin)
            self.kblock.grid.set_potential(self.kpoint.spin, self.local_op.potential)
            self.kblock.use_grid_potential(self.kpoint.spin)
        if getattr(self.kblock, "n_orb", 0):
            # the orbital block of D travels with the Hamiltonian too (a Noop Hubbard term is V = 0)
            self.kblock.set_orbital_coefficients(None if self.hubbard_op is None else self.hubbard_op.D)
        return self.kblock

    @property
    def shape(self):
        return (self.kpoint.n_G, self.kpoint.n_G)

    def mul(self, psi, out=None):
        """Hψ for a block of bands; psi: (n_bands, n_G) complex128 on the device."""
        return self.bind().apply_h(psi, out)

    __matmul__ = mul


class Hamiltonian:
    def __init__(self, basis, blocks):
        self.basis, self.blocks = basis, blocks

    def __getitem__(self, ik):
        return self.blocks[ik]

    def mul(self, psi):
        return [blk.mul(p) for blk, p in zip(self.blocks, psi)]

    __matmul__ = mul


KSUM_TERMS = ("Kinetic", "AtomicNonlocal", "Entropy")     # energies that are sums over the (k, spin) blocks


def ksum_energy_partials(basis, psi, occupation, eigenvalues, eF):
    """This rank's partial sums of the k-summed energy terms (kinetic.jl:54, nonlocal.jl:44, entropy.jl:39 before their
    mpi_sum): next_density packs them behind the density so that one allreduce serves compute_density and the energies."""
    names = [n for n in KSUM_TERMS if basis.term(n) is not None]
    basis._be_cache = {}
    try:
        from .terms import prefetch_band_energies
        prefetch_band_energies(basis, psi)
        vals = [basis.term(n).local_energy(basis, psi, occupation, eigenvalues=eigenvalues, eF=eF) for n in names]
    finally:
        basis._be_cache = None
    return names, np.array(vals, dtype=np.float64)


def _ksum_totals(basis, psi, occupation, eigenvalues, eF):
    """Totals over all ranks of the k-summed terms: taken from the step's packed allreduce when (psi, occupation) are the
    objects next_density produced, otherwise one packed allreduce here."""
    if psi is None or occupation is None:
        return {}
    c = getattr(basis, "_ksum_cache", None)
    if c is not None and c["psi"] is psi and c["occupation"] is occupation and c["eF"] == eF:
        return c["totals"]
    names, vals = ksum_energy_partials(basis, psi, occupation, eigenvalues, eF)
    if not np.all(np.isfinite(vals)):
        return dict(zip(names, vals))
    return dict(zip(names, basis.comm_kpts.allreduce(vals, "sum")))


def energy_hamiltonian(basis, psi, occupation, *, rho, eigenvalues=None, eF=None, hubbard_n=None, **kw):
    """Hamiltonian.jl:200-227: energies of every term + the per-k Hamiltonian blocks."""
    energies, per_term_ops = Energies(), []
    totals = _ksum_totals(basis, psi, occupation, eigenvalues, eF)
    for name, term in zip(basis.model.term_names, basis.terms):
        E, ops = term.ene_ops(basis, psi, occupation, rho=rho, eigenvalues=eigenvalues, eF=eF, ksum_total=totals.get(name),
                              hubbard_n=hubbard_n)
        energies[name] = E
        per_term_ops.append(ops)
    pot_cache = {}
    blocks = [DftHamiltonianBlock(basis, ik, [ops[ik] for ops in per_term_ops], pot_cache)
              for ik in range(len(basis.kpoints))]
    return energies, Hamiltonian(basis, blocks)


def energy(basis, psi, occupation, *, rho, eigenvalues=None, eF=None, hubbard_n=None, **kw):
    """Hamiltonian.jl:232-236 (energies only)."""
    energies = Energies()
    totals = _ksum_totals(basis, psi, occupation, eigenvalues, eF)
    for name, term in zip(basis.model.term_names, basis.terms):
        energies[name] = term.ene_ops(basis, psi, occupation, rho=rho, eigenvalues=eigenvalues, eF=eF,
                                      ksum_total=totals.get(name), hubbard_n=hubbard_n)[0]
    return energies
