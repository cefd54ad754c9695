"""Energy terms and their operators (host-side mirror of src/terms/*.jl for the DFT model:
Kinetic, AtomicLocal, AtomicNonlocal, Ewald, PspCorrection, Hartree, Xc, Entropy).

A term object exposes `ene_ops(basis, psi, occupation, rho=..., ...) -> (E, ops)` like
src/terms/terms.jl:6-12; operators are the RealFourierOperator kinds of src/terms/operators.jl.
Setup arithmetic (form factors, structure factors, Ewald) is vectorised torch on the device; the per-step
work on orbitals (kinetic / nonlocal band energies) goes through libdftk_b200.
"""
import math
import numpy as np
import torch
from scipy.special import erf, erfc

from . import xc as xcmod
from .pseudo import solid_harmonic_real, atom_decay_length
from .basis import estimate_integer_lattice_bounds
from .device import KBlock


# ------------------------------------------------------------------ operators (operators.jl)
class RealFourierOperator:
    pass


class NoopOperator(RealFourierOperator):
    def __init__(self, basis, kpoint):
        self.basis, self.kpoint = basis, kpoint


class RealSpaceMultiplication(RealFourierOperator):
    def __init__(self, basis, kpoint, potential):
        self.basis, self.kpoint, self.potential = basis, kpoint, potential


class FourierMultiplication(RealFourierOperator):
    def __init__(self, basis, kpoint, multiplier):
        self.basis, self.kpoint, self.multiplier = basis, kpoint, multiplier


class NonlocalOperator(RealFourierOperator):
    """`hubbard`: the operator Φ V Φ' of TermHubbard, whose columns the k-block carries beside the atomic projectors."""

    def __init__(self, basis, kpoint, P, D, hubbard=False):
        self.basis, self.kpoint, self.P, self.D, self.hubbard = basis, kpoint, P, D, hubbard


# ------------------------------------------------------------------ terms
def _xp(p):
    return torch if isinstance(p, torch.Tensor) else np


class BlowupIdentity:
    """kinetic.jl:63-67: the standard kinetic energy |p|²/2."""

    def __call__(self, p, Ecut):
        return _xp(p).ones_like(p)

    def __repr__(self):
        return "BlowupIdentity()"


class BlowupCHV:
    """kinetic.jl:70-95, the blow-up of arXiv:2210.00442: with x = |p| / sqrt(2 Ecut) the factor is 1 below x = 0.85,
    Ecut/Ekin · Ca/(1-x)² from x = 0.9 on, and a C^∞ interpolation of x² and Ca/(1-x)² in between, so that the bands
    become C² functions of k at a fixed cutoff (energy-cutoff smearing).  `p` is a NumPy array or a torch tensor."""
    x1, x2 = 0.85, 0.90
    Ca = 0.013952310177257383          # optimised to best match the x -> x² curve

    def __call__(self, p, Ecut):
        xp = _xp(p)
        x = p / math.sqrt(2 * Ecut)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = Ecut / (p ** 2 / 2)
            blow = self.Ca / (1 - x) ** 2
            t = (x - self.x1) / (self.x2 - self.x1)
            fa = xp.where(t > 0, xp.exp(-1 / xp.where(t > 0, t, 1.0)), 0.0)
            fb = xp.where(1 - t > 0, xp.exp(-1 / xp.where(1 - t > 0, 1 - t, 1.0)), 0.0)
            step = fa / (fa + fb)
            mid = ratio * ((1 - step) * x ** 2 + step * blow)
            return xp.where(x < self.x1, 1.0, xp.where(x < self.x2, mid, ratio * blow))

    def __repr__(self):
        return "BlowupCHV()"


class BlowupAbinit:
    """kinetic.jl:98-110, ABINIT's ecutsm: with Ecutsm = Ecutsm · Ecut the factor is 1 up to |p| = sqrt(2 (Ecut - Ecutsm))
    and 1 / (x² (3 + x - 6x² + 3x²)) of x = (Ecut - |p|²/2) / Ecutsm above (the reference's polynomial as written)."""

    def __init__(self, Ecutsm=0.5):
        self.Ecutsm = float(Ecutsm)

    def __call__(self, p, Ecut):
        xp = _xp(p)
        Ecutsm = Ecut * self.Ecutsm
        assert Ecutsm < Ecut
        x = (Ecut - p ** 2 / 2) / Ecutsm
        with np.errstate(divide="ignore"):
            return xp.where(p <= math.sqrt(2 * (Ecut - Ecutsm)), 1.0, 1 / (x ** 2 * (3 + x - 6 * x ** 2 + 3 * x ** 2)))

    def __repr__(self):
        return f"BlowupAbinit(Ecutsm={self.Ecutsm})"


class Kinetic:
    """kinetic.jl:7-12: the kinetic term with a scaling factor and a blow-up; a plain "Kinetic" is Kinetic()."""
    name = "Kinetic"

    def __init__(self, scaling_factor=1, blowup=None):
        self.scaling_factor = scaling_factor
        self.blowup = BlowupIdentity() if blowup is None else blowup

    def __call__(self, basis):
        return TermKinetic(basis, self.scaling_factor, self.blowup)

    def __repr__(self):
        return f"Kinetic(scaling_factor={self.scaling_factor}, blowup={self.blowup!r})"


class TermKinetic:
    """kinetic.jl:14-57: kinetic_energies[ik] = scaling_factor · |G+k|²/2 · blowup(|G+k|, Ecut), the table every device
    path (Hψ, the preconditioners, band energies) reads from the k-block."""

    def __init__(self, basis, scaling_factor=1.0, blowup=None):
        self.kinetic_energies = []
        for kpt in basis.kpoints:
            p = basis.Gplusk_vectors_cart(kpt)
            ekin = (scaling_factor * (p * p).sum(dim=1) / 2)
            if blowup is not None and not isinstance(blowup, BlowupIdentity):
                ekin = ekin * blowup(p.norm(dim=1), basis.Ecut)
            self.kinetic_energies.append(ekin.contiguous())

    def local_energy(self, basis, psi, occupation, **kw):
        """Σ over this rank's blocks (the mpi_sum of kinetic.jl:54 is done by the caller, packed with the other sums)."""
        E = 0.0
        for ik, kb in enumerate(basis.kblocks):
            both = _band_energies_shared(basis, ik, psi[ik])
            ek = both[0] if both is not None else _band_energies(kb, psi[ik], want_nl=False)[0]
            E += basis.kweights[ik] * float(np.sum(np.asarray(occupation[ik]) * ek))
        return E

    def ene_ops(self, basis, psi, occupation, ksum_total=None, **kw):
        ops = [FourierMultiplication(basis, k, self.kinetic_energies[ik]) for ik, k in enumerate(basis.kpoints)]
        if psi is None or occupation is None:
            return math.inf, ops
        if ksum_total is None:
            ksum_total = basis.comm_kpts.sum(self.local_energy(basis, psi, occupation))
        return float(ksum_total), ops


def _band_energies(kb, psik, want_nl=True, want_kin=True):
    import ctypes
    from ._lib import check
    from .device import _ptr
    nb = psik.shape[0]
    ek = np.zeros(nb) if want_kin else None
    en = np.zeros(nb) if want_nl else None
    check(kb.ctx.L.dftk_b200_band_energies(kb.h, _ptr(psik), nb, _ptr(ek), _ptr(en)), kb.ctx.h)
    return ek, en


def _band_energies_shared(basis, ik, psik):
    """Within one energy evaluation (energy_hamiltonian / energy set `basis._be_cache`) the kinetic and the nonlocal term
    need per-band energies of the same orbitals: one dftk_b200_band_energies call per k-block serves both."""
    cache = getattr(basis, "_be_cache", None)
    if cache is None or basis.term("Kinetic") is None or basis.term("AtomicNonlocal") is None:
        return None
    if ik not in cache:
        cache[ik] = _band_energies(basis.kblocks[ik], psik)
    return cache[ik]


def prefetch_band_energies(basis, psi):
    """All k-blocks of this rank in ONE library call (dftk_b200_band_energies_multi) into the evaluation's cache."""
    cache = getattr(basis, "_be_cache", None)
    if cache is None or basis.term("Kinetic") is None or basis.term("AtomicNonlocal") is None or len(cache):
        return
    from .device import band_energies_multi
    ek, en = band_energies_multi(basis.kblocks, [p.contiguous() for p in psi])
    for ik in range(len(basis.kblocks)):
        cache[ik] = (ek[ik], en[ik])


class TermAtomicLocal:
    """local.jl:108-138: V(G) = sum_atoms e^{-iG·r} v_loc(|G|)/sqrt(Ω), real-space via our own FFT."""

    def __init__(self, basis):
        model = basis.model
        pn = basis.G_vectors_cart.norm(dim=1)
        Gf = basis.G_vectors.to(torch.float64)
        pot = torch.zeros(basis.N, dtype=torch.complex128, device=pn.device)
        for group in model.atom_groups:
            ff = model.atoms[group[0]].psp.eval_psp_local_fourier(pn)
            sf = structure_factor(basis, [model.positions[i] for i in group])     # Σ_a e^{-2πi G·r_a}, one kernel
            pot += sf * ff / math.sqrt(model.unit_cell_volume)
        self.potential_values = basis.irfft(basis.enforce_real(pot)).reshape(-1)

    def ene_ops(self, basis, psi, occupation, rho=None, **kw):
        ops = [RealSpaceMultiplication(basis, k, self.potential_values) for k in basis.kpoints]
        E = math.inf if rho is None else float((rho.sum(dim=0) * self.potential_values).sum() * basis.dvol)
        return E, ops


def structure_factor(basis, positions, coefficients=None):
    """Σ_a c_a exp(-2πi G·r_a) on the whole FFT cube: one fused kernel over (cube point, atom)
    (dftk_b200_structure_factor) instead of chunked N × n_atoms phase tables."""
    from ._lib import check
    from .device import _ptr
    ctx = basis.architecture.ctx
    pos = np.ascontiguousarray(np.array([np.asarray(p, dtype=np.float64) for p in positions]))
    cf = None if coefficients is None else np.ascontiguousarray(coefficients, dtype=np.float64)
    out = torch.empty(basis.N, dtype=torch.complex128, device=ctx.device)
    check(ctx.L.dftk_b200_structure_factor(basis.fft_grid.h, len(pos), _ptr(pos), _ptr(cf), _ptr(out)), ctx.h)
    return out


def build_projection_coefficients(psp):
    """nonlocal.jl:128-141: block diagonal over (l, m) with psp.h[l] blocks."""
    n = psp.count_n_proj()
    D = np.zeros((n, n))
    c = 0
    for l in range(psp.lmax + 1):
        for _ in range(2 * l + 1):
            k = psp.count_n_proj_radial(l)
            D[c:c + k, c:c + k] = psp.h[l]
            c += k
    return D


def build_projector_form_factors(psp, Gpk_cart):
    """nonlocal.jl:205-244; (n_proj, n_G) complex, ordering (l, m, i)."""
    pn = Gpk_cart.norm(dim=1)
    rows = []
    for l in range(psp.lmax + 1):
        radial = [psp.eval_psp_projector_fourier(i, l, pn) for i in range(1, psp.count_n_proj_radial(l) + 1)]
        for m in range(-l, l + 1):
            ang = solid_harmonic_real(l, m, Gpk_cart).to(torch.complex128) * ((-1j) ** l)
            rows += [r * ang for r in radial]
    if not rows:
        return torch.zeros((0, Gpk_cart.shape[0]), dtype=torch.complex128, device=Gpk_cart.device)
    return torch.stack(rows, dim=0)


class TermAtomicNonlocal:
    """nonlocal.jl:9-47,107-199.  P is stored as (n_proj, n_G) = column-major n_G × n_proj."""

    def __init__(self, basis):
        model = basis.model
        self.ops = []
        cache = {}
        for kpt in basis.kpoints:
            key = id(kpt.mapping)
            if key not in cache:
                Gpk = basis.Gplusk_vectors(kpt)
                Gpk_cart = basis.Gplusk_vectors_cart(kpt)
                from ._lib import check
                from .device import _ptr
                ctx = basis.architecture.ctx
                Ds = []
                n_rows_total = sum(len(g) * model.atoms[g[0]].psp.count_n_proj() for g in model.atom_groups)
                P = torch.empty((n_rows_total, kpt.n_G), dtype=torch.complex128, device=Gpk.device) if n_rows_total else None
                gpk_t = Gpk.T.contiguous()                               # (3, n_pw) reduced G+k, component-major
                row = 0
                for group in model.atom_groups:
                    psp = model.atoms[group[0]].psp
                    ff = (build_projector_form_factors(psp, Gpk_cart) / math.sqrt(model.unit_cell_volume)).contiguous()
                    Dat = build_projection_coefficients(psp)
                    nr = ff.shape[0]
                    if nr:
                        # P[(a, p), G] = e^{-2πi (G+k)·r_a} ff[p, G] for all atoms of the species: one fused kernel
                        pos = np.ascontiguousarray(np.array([model.positions[ia] for ia in group], dtype=np.float64))
                        check(ctx.L.dftk_b200_build_projectors(ctx.h, kpt.n_G, _ptr(gpk_t), len(group), _ptr(pos), nr, _ptr(ff),
                                                               _ptr(P[row:row + nr * len(group)])), ctx.h)
                        row += nr * len(group)
                    Ds += [Dat] * len(group)
                n = sum(d.shape[0] for d in Ds)
                D = np.zeros((n, n))
                o = 0
                for d in Ds:
                    D[o:o + d.shape[0], o:o + d.shape[0]] = d
                    o += d.shape[0]
                cache[key] = (P, D)
            P, D = cache[key]
            self.ops.append(NonlocalOperator(basis, kpt, P, D))

    def local_energy(self, basis, psi, occupation, **kw):
        E = 0.0
        for ik, kb in enumerate(basis.kblocks):
            both = _band_energies_shared(basis, ik, psi[ik])
            en = both[1] if both is not None else _band_energies(kb, psi[ik], want_kin=False)[1]
            E += basis.kweights[ik] * float(np.sum(en * np.asarray(occupation[ik])))
        return E

    def ene_ops(self, basis, psi, occupation, ksum_total=None, **kw):
        if psi is None or occupation is None:
            return math.inf, self.ops
        if ksum_total is None:
            ksum_total = basis.comm_kpts.sum(self.local_energy(basis, psi, occupation))
        return float(ksum_total), self.ops


def energy_ewald(lattice, charges, positions, eta=None):
    """ewald.jl:40-168 (energy only)."""
    charges = np.asarray(charges, dtype=float)
    pos = np.array([np.asarray(p, dtype=float) for p in positions])
    recip = 2 * math.pi * np.linalg.inv(lattice.T)
    if eta is None:
        eta = math.sqrt(math.sqrt(1.69 * np.linalg.norm(recip / (2 * math.pi)) / np.linalg.norm(lattice))) / 2
    max_exp = -math.log(np.finfo(float).eps) + 5
    Glims = estimate_integer_lattice_bounds(recip, math.sqrt(max_exp) * 2 * eta)
    poslims = [float(np.max(pos[:, i][:, None] - pos[:, i][None, :])) for i in range(3)]
    Rlims = estimate_integer_lattice_bounds(lattice, math.sqrt(max_exp) / eta, poslims)
    vol = abs(np.linalg.det(lattice))
    G = np.stack(np.meshgrid(*[np.arange(-g, g + 1) for g in Glims], indexing="ij"), -1).reshape(-1, 3)
    G = G[np.any(G != 0, axis=1)]
    Gsq = np.sum((G @ recip.T) ** 2, axis=1)
    sum_recip = -(charges.sum() ** 2 / (4 * eta ** 2))
    cs = np.zeros(len(G)); sn = np.zeros(len(G))
    for c in range(0, len(pos), 32):
        ph = 2 * math.pi * (G @ pos[c:c + 32].T)
        cs += (np.cos(ph) * charges[c:c + 32]).sum(axis=1)
        sn += (np.sin(ph) * charges[c:c + 32]).sum(axis=1)
    sum_recip += np.sum((cs ** 2 + sn ** 2) * np.exp(-Gsq / (4 * eta ** 2)) / Gsq)
    sum_recip *= 4 * math.pi / vol
    sum_real = -2 * eta / math.sqrt(math.pi) * np.sum(charges ** 2)
    R = np.stack(np.meshgrid(*[np.arange(-g, g + 1) for g in Rlims], indexing="ij"), -1).reshape(-1, 3).astype(float)
    Rcart = R @ lattice.T
    nonzero = np.any(R != 0, axis=1)
    for i in range(len(pos)):
        d = (pos[i] - pos) @ lattice.T                       # (n_atoms, 3)
        dist = np.linalg.norm(d[:, None, :] - Rcart[None, :, :], axis=2)   # (n_atoms, n_R)
        mask = np.ones_like(dist, dtype=bool)
        mask[i, ~nonzero] = False
        zz = charges[i] * charges[:, None] * np.ones_like(dist)
        sum_real += np.sum(zz[mask] * erfc(eta * dist[mask]) / dist[mask])
    return (sum_recip + sum_real) / 2


class TermEwald:
    def __init__(self, basis):
        from .forces import energy_forces_ewald_device
        m = basis.model
        self.energy = energy_forces_ewald_device(basis.architecture.ctx, m.lattice, [a.charge_ionic() for a in m.atoms],
                                                 m.positions)[0]

    def ene_ops(self, basis, psi, occupation, **kw):
        return self.energy, [NoopOperator(basis, k) for k in basis.kpoints]


class TermPspCorrection:
    """psp_correction.jl:26-35."""

    def __init__(self, basis):
        m = basis.model
        corr = sum(len(g) * m.atoms[g[0]].psp.eval_psp_energy_correction() for g in m.atom_groups)
        self.energy = corr * sum(a.n_elec_valence() for a in m.atoms) / m.unit_cell_volume

    def ene_ops(self, basis, psi, occupation, **kw):
        return self.energy, [NoopOperator(basis, k) for k in basis.kpoints]


class TermHartree:
    """hartree.jl:29-59."""

    def __init__(self, basis):
        G2 = (basis.G_vectors_cart ** 2).sum(dim=1)
        g = 4 * math.pi / torch.where(G2 == 0, torch.ones_like(G2), G2)
        g[0] = 0.0
        self.poisson_green_coeffs = basis.enforce_real(g)

    def ene_ops(self, basis, psi, occupation, rho=None, **kw):
        rf = basis.fft(rho.sum(dim=0)).reshape(-1)
        pf = self.poisson_green_coeffs * rf
        pot = basis.irfft(pf).reshape(-1)
        E = float(torch.real(torch.vdot(pf, rf)) / 2)
        return E, [RealSpaceMultiplication(basis, k, pot) for k in basis.kpoints]


def core_density(basis):
    """ρcore of the non-linear core correction (xc.jl:30-40): the superposition of the model core densities of every
    species that has one, split equally over the spin components (ρ_from_total), not renormalised.  None if no species
    has a core density."""
    model = basis.model
    groups = [g for g in model.atom_groups if getattr(model.atoms[g[0]].psp, "has_core_density", False)]
    if not groups:
        return None
    pn = basis.G_vectors_cart.norm(dim=1)
    rho = torch.zeros(basis.N, dtype=torch.complex128, device=pn.device)
    for group in groups:
        ff = model.atoms[group[0]].psp.eval_psp_core_density_fourier(pn)
        rho += structure_factor(basis, [model.positions[i] for i in group]) * ff / math.sqrt(model.unit_cell_volume)
    rtot = basis.irfft(basis.enforce_real(rho)).reshape(-1)
    n_spin = model.n_spin_components
    return (rtot[None, :] if n_spin == 1 else torch.stack([rtot / 2, rtot / 2])).contiguous()


class TermXc:
    """xc.jl:84-160 (LDA / GGA; potential = Vρ - 2 ∇·(Vσ ∇ρ)).  With a model core density (NLCC) the energy and the
    potential are evaluated at ρ + ρcore (gradients included); the potential is still the derivative with respect to ρ."""

    def __init__(self, basis):
        self.functionals = list(basis.model.functionals)
        self.rho_core = core_density(basis)

    def potential(self, basis, rho):
        if self.rho_core is not None:
            rho = rho + self.rho_core
        n_spin = rho.shape[0]
        is_gga = any(f.startswith("gga") for f in self.functionals)
        sigma = grad = None
        Gc = basis.G_vectors_cart
        if is_gga:
            rf = basis.fft(rho)                                        # (n_spin, N)
            grad = torch.stack([basis.irfft(1j * Gc[:, a][None, :] * rf) for a in range(3)], dim=1)  # (s,3,N)
            if n_spin == 1:
                sigma = (grad[0] * grad[0]).sum(dim=0)[None, :]
            else:
                sigma = torch.stack([(grad[0] * grad[0]).sum(0), (grad[0] * grad[1]).sum(0), (grad[1] * grad[1]).sum(0)])
        e, vr, vs = xcmod.evaluate(basis.architecture.ctx, self.functionals, rho, sigma)
        E = float(e.sum() * basis.dvol)
        pot = vr.clone()
        if is_gga:
            ts = (lambda s, t: 0) if n_spin == 1 else (lambda s, t: (0, 1, 1, 2)[2 * s + t])
            for s in range(n_spin):
                gsum = torch.zeros(basis.N, dtype=torch.complex128, device=rho.device)
                for a in range(3):
                    op = sum((1.0 if s == t else 0.5) * vs[ts(s, t)] * grad[t, a] for t in range(n_spin))
                    gsum += 1j * Gc[:, a] * basis.fft(op).reshape(-1)
                pot[s] += -2 * basis.irfft(gsum).reshape(-1)
        return E, pot

    def ene_ops(self, basis, psi, occupation, rho=None, **kw):
        E, pot = self.potential(basis, rho)
        return E, [RealSpaceMultiplication(basis, k, pot[k.spin]) for k in basis.kpoints]


def methfessel_paxton_order(kind):
    """The order n of a ("MethfesselPaxton", n) smearing, None for every other kind."""
    if isinstance(kind, (tuple, list)) and len(kind) == 2 and kind[0] == "MethfesselPaxton":
        return kind[1]
    return None


def _mp_sums(n, x):
    """Smearing.jl:133-168 for all of x at once: the A(i) H_k(x) sums of the Methfessel-Paxton occupation, entropy and
    derivative, from the physicists' Hermite recursion H_k = 2x H_{k-1} - 2(k-1) H_{k-2} evaluated up to H_{2n}."""
    H = [np.ones_like(x), 2 * x]
    for k in range(2, 2 * n + 1):
        H.append(2 * x * H[k - 1] - 2 * (k - 1) * H[k - 2])
    A = [(-1) ** i / (math.factorial(i) * 4 ** i * math.sqrt(math.pi)) for i in range(n + 1)]
    occ = sum((A[i] * H[2 * i - 1] for i in range(1, n + 1)), np.zeros_like(x))
    ent = sum(A[i] * (H[2 * i] / 2 + (2 * i * H[2 * i - 2] if i else 0)) for i in range(n + 1))
    der = sum(A[i] * H[2 * i] for i in range(n + 1))
    return occ, ent, der


_MV_SHIFT = 1 / math.sqrt(2)


def smearing_occupation(kind, x):
    """Smearing.occupation (Smearing.jl): f(x) with x = (ε - εF) / T; 1 at -∞ and 0 at +∞ for every kind."""
    x = np.asarray(x, dtype=float)
    if kind == "None":
        return np.where(x > 0, 0.0, 1.0)
    if kind == "FermiDirac":
        ex = np.exp(-np.abs(x))
        return np.where(x > 0, ex / (1 + ex), 1 / (1 + ex))
    if kind == "Gaussian":
        return erfc(x) / 2
    if kind == "MarzariVanderbilt":
        u = x + _MV_SHIFT
        return -erf(u) / 2 + np.exp(-u ** 2) / math.sqrt(2 * math.pi) + 0.5
    n = methfessel_paxton_order(kind)
    if n is not None:
        xf = np.where(np.isinf(x), 0.0, x)
        f = erfc(xf) / 2 + _mp_sums(n, xf)[0] * np.exp(-xf ** 2)
        return np.where(np.isinf(x), np.where(x > 0, 0.0, 1.0), f)
    raise NotImplementedError(kind)


def smearing_entropy(kind, x):
    """Smearing.entropy: s(x) with s'(x) = x f'(x)."""
    x = np.asarray(x, dtype=float)
    if kind == "None":
        return np.zeros_like(x)
    if kind == "FermiDirac":
        f = smearing_occupation(kind, x)
        eps = np.finfo(float).eps
        out = np.zeros_like(x)
        ok = (np.abs(f) >= eps) & (np.abs(1 - f) >= eps)
        out[ok] = -(f[ok] * np.log(f[ok]) + (1 - f[ok]) * np.log(1 - f[ok]))
        return out
    if kind == "Gaussian":
        return np.exp(-x ** 2) / (2 * math.sqrt(math.pi))
    if kind == "MarzariVanderbilt":
        u = x + _MV_SHIFT
        return u * np.exp(-u ** 2) / math.sqrt(2 * math.pi)
    n = methfessel_paxton_order(kind)
    if n is not None:
        return _mp_sums(n, x)[1] * np.exp(-x ** 2)
    raise NotImplementedError(kind)


def occupation_derivative(kind, x):
    """Smearing.occupation_derivative in closed form: f'(x), an approximation of minus the delta function."""
    x = np.asarray(x, dtype=float)
    if kind == "None":
        return np.zeros_like(x)
    if kind == "FermiDirac":
        ex = np.exp(-np.abs(x))
        return -ex / (1 + ex) ** 2
    if kind == "Gaussian":
        return -np.exp(-x ** 2) / math.sqrt(math.pi)
    if kind == "MarzariVanderbilt":
        u = x + _MV_SHIFT
        return -np.exp(-u ** 2) * (2 + math.sqrt(2) * x) / math.sqrt(math.pi)
    n = methfessel_paxton_order(kind)
    if n is not None:            # f' = -Σ_i A(i) H_2i(x) e^{-x²}, the order-n Hermite expansion of -δ
        return -_mp_sums(n, x)[2] * np.exp(-x ** 2)
    raise NotImplementedError(kind)


class TermEntropy:
    """entropy.jl:11-42."""

    def __init__(self, basis):
        pass

    def local_energy(self, basis, psi, occupation, eigenvalues=None, eF=None, **kw):
        m = basis.model
        if m.temperature == 0:
            return 0.0
        if eigenvalues is None or eF is None:
            return math.inf
        E = 0.0
        for ik in range(len(basis.kpoints)):
            nb = psi[ik].shape[0]
            E -= (m.temperature * basis.kweights[ik] * m.filled_occupation
                  * float(np.sum(smearing_entropy(m.smearing, (np.asarray(eigenvalues[ik])[:nb] - eF) / m.temperature))))
        return E

    def ene_ops(self, basis, psi, occupation, eigenvalues=None, eF=None, ksum_total=None, **kw):
        ops = [NoopOperator(basis, k) for k in basis.kpoints]
        m = basis.model
        if m.temperature == 0:
            return 0.0, ops
        if psi is None or occupation is None or eigenvalues is None or eF is None:
            return math.inf, ops
        if ksum_total is None:
            ksum_total = basis.comm_kpts.sum(self.local_energy(basis, psi, occupation, eigenvalues=eigenvalues, eF=eF))
        return float(ksum_total), ops


_TERMS = dict(Kinetic=TermKinetic, AtomicLocal=TermAtomicLocal, AtomicNonlocal=TermAtomicNonlocal,
              Ewald=TermEwald, PspCorrection=TermPspCorrection, Hartree=TermHartree, Xc=TermXc,
              Entropy=TermEntropy)


def instantiate(name, basis):
    if not isinstance(name, str):          # a term object such as Hubbard(...): called with the basis (hubbard.jl:119)
        return name(basis)
    if name not in _TERMS:
        raise NotImplementedError(f"term {name} is outside the hot-path scope of dftk_b200")
    return _TERMS[name](basis)


def build_kblocks(basis):
    """One device k-block per (k, spin): kin from Kinetic, P/D from AtomicNonlocal, the orbital columns from Hubbard."""
    kin_t, nl_t, hub_t = basis.term("Kinetic"), basis.term("AtomicNonlocal"), basis.term("Hubbard")
    out = []
    for ik, kpt in enumerate(basis.kpoints):
        kin = kin_t.kinetic_energies[ik] if kin_t is not None else None
        P = D = None
        if nl_t is not None and nl_t.ops[ik].P is not None:
            P, D = nl_t.ops[ik].P, nl_t.ops[ik].D
        out.append(KBlock(basis.fft_grid, kpt.mapping.cpu().numpy(), kin=kin, P=P, D=D, spin=kpt.spin,
                          kweight=basis.kweights[ik]))
        if hub_t is not None:
            out[-1].set_orbitals(hub_t.P_vec[ik])
    return out


def guess_density(basis, magnetic_moments=None):
    """density_methods.jl:103-181,237-244 with ValenceDensityAuto: superposition of atomic valence densities, the
    pseudo-atomic one (PP_RHOATOM) for species whose pseudopotential has it, a Gaussian for every other species."""
    model = basis.model
    pn = basis.G_vectors_cart.norm(dim=1)
    Gf = basis.G_vectors.to(torch.float64)
    form_factors = {}

    def form_factor(a0):
        if a0 not in form_factors:
            if getattr(a0.psp, "has_valence_density", False):
                form_factors[a0] = a0.psp.eval_psp_valence_density_fourier(pn)
            else:
                L = atom_decay_length(a0.n_elec_core(), a0.n_elec_valence())
                form_factors[a0] = a0.charge_ionic() * torch.exp(-(pn * L) ** 2)
        return form_factors[a0]

    def superposition(coeffs):
        rho = torch.zeros(basis.N, dtype=torch.complex128, device=pn.device)
        for group in model.atom_groups:
            ff = form_factor(model.atoms[group[0]])
            sf = structure_factor(basis, [model.positions[i] for i in group], [coeffs[i] for i in group])
            rho += sf * ff / math.sqrt(model.unit_cell_volume)
        return basis.irfft(basis.enforce_real(rho)).reshape(-1)

    rtot = superposition([1.0] * len(model.atoms))
    if model.n_spin_components == 1:
        rho = rtot[None, :]
    else:
        mm = magnetic_moments if magnetic_moments is not None else model.magnetic_moments
        coeffs = [m / a.n_elec_valence() for m, a in zip(mm, model.atoms)]
        rspin = superposition(coeffs) if any(c != 0 for c in coeffs) else torch.zeros_like(rtot)
        rho = torch.stack([(rtot + rspin) / 2, (rtot - rspin) / 2])
    Nel = float(rho.sum() * basis.dvol)
    if Nel > 0:
        rho = rho * (model.n_electrons / Nel)
    return rho.contiguous()
