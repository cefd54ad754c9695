"""PlaneWaveBasis / Kpoint / MonkhorstPack (host-side mirror of src/PlaneWaveBasis.jl:129-369,
src/Kpoint.jl:6-74, src/bzmesh.jl:41-95, src/fft.jl:231-337).  Setup code; heavy arrays are torch
tensors on the GPU, every transform goes through libdftk_b200's own FFT kernels."""
import math
from fractions import Fraction
import numpy as np
import torch

from .model import SymOp, SYMMETRY_TOLERANCE
from .device import FFTGrid, KBlock
from .parallel import KpointComm, BlockLayout, pad_kpoints_for_ranks


# ------------------------------------------------------------------ grid sizes (fft.jl:231-337)
def _is_smooth(n, primes=(2, 3, 5)):
    for p in primes:
        while n % p == 0:
            n //= p
    return n == 1


def next_compatible_fft_size(size, factors=(1,)):
    f = int(np.prod(factors))
    while not (size % f == 0 and _is_smooth(size)):
        size += 1
    return size


def estimate_integer_lattice_bounds(M, delta, shift=(0, 0, 0), tol=math.sqrt(np.finfo(float).eps)):
    inv_t = np.linalg.inv(M.T)
    lims = [np.linalg.norm(inv_t[:, i]) * delta + shift[i] for i in range(3)]
    return [0 if x == 0 else int(math.ceil(x - tol)) for x in lims]


def compute_fft_size(model, Ecut, supersampling=2.0, factors=(1,)):
    Glims = estimate_integer_lattice_bounds(model.recip_lattice, supersampling * math.sqrt(2 * Ecut))
    return tuple(next_compatible_fft_size(2 * g + 1, factors) for g in Glims)


def G_axis(n):
    stop, start = (n - 1) // 2, -(n // 2)
    return np.array(list(range(0, stop + 1)) + list(range(start, 0)), dtype=np.int64)


# ------------------------------------------------------------------ k-grids (bzmesh.jl)
def normalize_kpoint_coordinate(k):
    k = np.asarray(k, dtype=float)
    k = k - np.floor(k + 0.5)
    return np.where(k >= 0.5, k - 1.0, k)


class MonkhorstPack:
    def __init__(self, kgrid_size, kshift=(0, 0, 0)):
        self.kgrid_size = tuple(int(x) for x in kgrid_size)
        self.kshift = tuple(Fraction(x).limit_denominator(2) for x in kshift)
        for s in self.kshift:
            if s not in (0, Fraction(1, 2)):
                raise ValueError("Only kshifts of 0 or 1//2 implemented.")

    def reducible_kcoords(self):
        ks = np.array(self.kgrid_size)
        start = -np.floor((ks - 1) / 2).astype(int)
        stop = np.ceil((ks - 1) / 2).astype(int)
        sh = np.array([float(s) for s in self.kshift])
        return [normalize_kpoint_coordinate((sh + np.array([i, j, k])) / ks)
                for k in range(start[2], stop[2] + 1) for j in range(start[1], stop[1] + 1)
                for i in range(start[0], stop[0] + 1)]

    def __len__(self):
        return int(np.prod(self.kgrid_size))


class ExplicitKpoints:
    def __init__(self, kcoords, kweights=None):
        self.kcoords = [np.array(k, dtype=float) for k in kcoords]
        self.kweights = list(kweights) if kweights is not None else [1.0 / len(kcoords)] * len(kcoords)
        if len(self.kcoords) != len(self.kweights):
            raise ValueError("kcoords and kweights need the same length")
        if abs(sum(self.kweights) - 1) > 1e-10:
            raise ValueError("kweights need to sum to 1")

    def reducible_kcoords(self):
        return self.kcoords


def _kkey(k):
    return tuple(np.round(normalize_kpoint_coordinate(k) * 1e6).astype(np.int64) % 1000000)


def irreducible_kcoords(kgrid, symmetries):
    """bzmesh.jl:55-95 (the spglib mesh reduction done by explicit orbit search; no time reversal)."""
    if isinstance(kgrid, ExplicitKpoints):
        return kgrid.kcoords, kgrid.kweights
    kall = kgrid.reducible_kcoords()
    index = {_kkey(k): i for i, k in enumerate(kall)}
    rep = -np.ones(len(kall), dtype=int)
    kirr, counts = [], []
    for i, k in enumerate(kall):
        if rep[i] >= 0:
            continue
        rep[i] = len(kirr)
        cnt = 1
        for op in symmetries:
            j = index.get(_kkey(op.S @ k))
            if j is not None and rep[j] < 0:
                rep[j] = len(kirr)
                cnt += 1
        kirr.append(k)
        counts.append(cnt)
    return kirr, [c / len(kall) for c in counts]


class Kpoint:
    """src/Kpoint.jl:6-18.  mapping is 0-based here (Julia: 1-based)."""

    def __init__(self, spin, coordinate, mapping, G_vectors):
        self.spin = spin
        self.coordinate = np.array(coordinate, dtype=float)
        self.mapping = mapping            # torch int64 (device), ascending
        self.G_vectors = G_vectors        # torch int64 (n_G, 3) device

    @property
    def n_G(self):
        return int(self.mapping.numel())


class PlaneWaveBasis:
    def __init__(self, model, *, Ecut, kgrid=(1, 1, 1), kshift=(0, 0, 0), fft_size=None, supersampling=2.0,
                 architecture=None, comm_kpts=None, comm_slab=None, use_symmetries_for_kpoint_reduction=True,
                 variational=True, _symmetries_respect_rgrid=None):
        """`comm_kpts`: shard the (k, spin) blocks over the ranks (the reference's only distribution).
        `comm_slab`: instead, let ALL ranks work on every k-block together (single-k multi-GPU, e.g. a Γ-only supercell):
        the eigensolver cuts the plane-wave rows into one slab per rank (dftk_b200_lobpcg_slab), compute_density splits
        the bands; everything else runs replicated on identical data.
        `_symmetries_respect_rgrid` (private): keep another basis's decision whether the symmetries must map the real-space
        grid onto itself, although `fft_size` is passed (unfold_bz); None: True exactly when `fft_size` is None."""
        from .architecture import B200
        if not variational:
            raise NotImplementedError("Non-variational calculations are not supported")
        self.model = model
        self.Ecut = float(Ecut)
        self.comm_kpts = comm_kpts or KpointComm()
        self.comm_slab = comm_slab if (comm_slab is not None and comm_slab.nranks > 1) else None
        if self.comm_slab is not None and self.comm_kpts.nranks > 1:
            raise NotImplementedError("comm_kpts and comm_slab cannot be combined yet: choose one distribution")
        dist_comm = self.comm_slab or (self.comm_kpts if self.comm_kpts.nranks > 1 else None)
        self.architecture = architecture or B200(comm=dist_comm)
        if self.comm_slab is not None and getattr(self.architecture.ctx, "nranks", 1) != self.comm_slab.nranks:
            raise ValueError("comm_slab needs an architecture whose context spans the same ranks (B200(comm=comm_slab))")
        dev = self.architecture.device
        self.kgrid = kgrid if isinstance(kgrid, (MonkhorstPack, ExplicitKpoints)) else MonkhorstPack(kgrid, kshift)
        symmetries_respect_rgrid = fft_size is None if _symmetries_respect_rgrid is None else bool(_symmetries_respect_rgrid)
        self.symmetries_respect_rgrid = symmetries_respect_rgrid
        if fft_size is None:
            dens = {Fraction(float(wi)).limit_denominator(12).denominator for s in model.symmetries for wi in s.w}
            factors = tuple(sorted({2, 3, 4, 6} & dens)) or (1,)
            fft_size = compute_fft_size(model, Ecut, supersampling, factors)
        self.fft_size = tuple(int(n) for n in fft_size)
        nx, ny, nz = self.fft_size
        max_E = float(np.sum((model.recip_lattice @ np.floor(np.array(self.fft_size) / 2)) ** 2) / 2)
        if Ecut > max_E:
            import warnings
            warnings.warn(f"For a variational method, Ecut should be less than the maximal kinetic energy "
                          f"the grid supports ({max_E})")
        self.N = nx * ny * nz
        self.dvol = model.unit_cell_volume / self.N
        self.ifft_normalization = 1 / math.sqrt(model.unit_cell_volume)
        self.fft_normalization = math.sqrt(model.unit_cell_volume) / self.N
        # symmetries compatible with the grids (symmetry.jl:162-205)
        syms = list(model.symmetries)
        if symmetries_respect_rgrid:
            n = np.array(self.fft_size)
            syms = [s for s in syms if np.all(np.abs(s.w * n - np.round(s.w * n)) / n <= SYMMETRY_TOLERANCE)]
        if isinstance(self.kgrid, MonkhorstPack):
            keys = {_kkey(k) for k in self.kgrid.reducible_kcoords()}
            ks, sh = np.array(self.kgrid.kgrid_size), np.array([float(s) for s in self.kgrid.kshift])
            probes = [(sh + np.array(d)) / ks for d in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1))]
            syms = [s for s in syms if all(_kkey(s.S @ p) in keys for p in probes)]
        self.symmetries = syms
        self.use_symmetries_for_kpoint_reduction = use_symmetries_for_kpoint_reduction
        if use_symmetries_for_kpoint_reduction:
            kcoords, kweights = irreducible_kcoords(self.kgrid, syms)
        else:
            kcoords, kweights = irreducible_kcoords(self.kgrid, [SymOp(np.eye(3), np.zeros(3))])
        self.n_irreducible_kpoints = len(kcoords)
        # (k, spin) block sharding.  The reference splits the k-points into contiguous chunks and keeps both spins of a
        # k-point on one rank (PlaneWaveBasis.jl:184-229); here the blocks b = ik + spin * n_kpt are flattened and dealt
        # to the ranks longest-first by cost ~ n_pw (SURVEY §8e), so spin x k fills all 8 GPUs of a box.
        comm = self.comm_kpts
        n_spin = model.n_spin_components
        kcoords, kweights = pad_kpoints_for_ranks(kcoords, kweights, comm.nranks, n_spin)
        self.kcoords_global = [np.array(k, dtype=float) for k in kcoords]
        self.kweights_global = list(kweights)
        n_kpt = len(kcoords)
        # device grid tables
        self.fft_grid = FFTGrid(self.architecture.ctx, self.fft_size, model.unit_cell_volume)
        gx, gy, gz = (torch.as_tensor(G_axis(n), device=dev) for n in self.fft_size)
        Z, Y, X = torch.meshgrid(gz, gy, gx, indexing="ij")
        self.G_vectors = torch.stack([X.reshape(-1), Y.reshape(-1), Z.reshape(-1)], dim=1)     # (N,3) int64
        self._recip = torch.as_tensor(model.recip_lattice, device=dev)
        Gf = self.G_vectors.to(torch.float64)
        self.G_vectors_cart = Gf @ self._recip.T

        sphere = self.sphere_mask
        costs = [1.0] * (n_kpt * n_spin)
        if comm.nranks > 1:          # every rank counts every sphere: the block -> rank map is identical everywhere
            npw = [float(sphere(k).sum().item()) for k in self.kcoords_global]
            costs = [npw[b % n_kpt] for b in range(n_kpt * n_spin)]
        self.layout = BlockLayout(n_kpt, n_spin, self.kweights_global, costs, comm.nranks, comm.rank)
        self.krange_thisproc_allspin = list(self.layout.mine)
        # k-blocks of this rank, spin-major then k
        self.kpoints, self.kweights = [], []
        base = {}
        for b in self.layout.mine:
            i, spin = b % n_kpt, b // n_kpt
            if i not in base:
                mapping = torch.nonzero(sphere(self.kcoords_global[i])).reshape(-1)
                base[i] = (mapping, self.G_vectors[mapping])
            mapping, Gk = base[i]
            self.kpoints.append(Kpoint(spin, self.kcoords_global[i], mapping, Gk))
            self.kweights.append(self.kweights_global[i])
        total_w = comm.sum(sum(self.kweights))
        assert abs(total_w - n_spin) < 1e-10
        # instantiate terms (PlaneWaveBasis.jl:256-259), then the device k-blocks
        from . import terms as _terms
        self.terms = [_terms.instantiate(name, self) for name in model.term_types]
        self.kblocks = _terms.build_kblocks(self)

    # ------------------------------------------------------------------ helpers
    def sphere_mask(self, kcoord):
        """Kpoint.jl:20-41: membership of every cube G in the kinetic-energy sphere of k-point `kcoord`."""
        p = (self.G_vectors.to(torch.float64) + torch.as_tensor(kcoord, device=self.G_vectors.device)) @ self._recip.T
        return (p * p).sum(dim=1) / 2 <= self.Ecut

    def Gplusk_vectors(self, kpt):
        return kpt.G_vectors.to(torch.float64) + torch.as_tensor(kpt.coordinate, device=kpt.G_vectors.device)

    def Gplusk_vectors_cart(self, kpt):
        return self.Gplusk_vectors(kpt) @ self._recip.T

    def term(self, name):
        for n, t in zip(self.model.term_names, self.terms):
            if n == name:
                return t
        return None

    def weighted_ksum(self, values):
        """PlaneWaveBasis.jl:509-512."""
        return self.comm_kpts.sum(sum(w * v for w, v in zip(self.kweights, values)))

    # cube FFTs on (n_spin|batch, N) arrays, src/fft.jl:106-109,155-161 -- own kernels
    def fft(self, f_real):
        f = f_real.to(torch.complex128).contiguous().clone()
        self.fft_grid.fft_cube(f.reshape(-1, self.N), -1)
        return f * self.fft_normalization

    def ifft(self, f_fourier):
        f = f_fourier.to(torch.complex128).contiguous().clone()
        self.fft_grid.fft_cube(f.reshape(-1, self.N), +1)
        return f * self.ifft_normalization

    def irfft(self, f_fourier):
        return self.ifft(f_fourier).real.contiguous()

    def index_G_vectors(self, G):
        """Linear cube index of integer G (…,3) or -1 if outside (PlaneWaveBasis.jl:465-480)."""
        n = torch.as_tensor(self.fft_size, device=G.device)
        start, stop = -(n // 2), (n - 1) // 2
        ok = ((G >= start) & (G <= stop)).all(dim=-1)
        i3 = torch.remainder(G, n)
        lin = i3[..., 0] + n[0] * (i3[..., 1] + n[1] * i3[..., 2])
        return torch.where(ok, lin, torch.full_like(lin, -1))

    def enforce_real(self, coeffs):
        """symmetry.jl:550-552: drop G whose -G is not on the grid."""
        if not hasattr(self, "_real_mask"):
            self._real_mask = self.index_G_vectors(-self.G_vectors) >= 0
        return torch.where(self._real_mask, coeffs, torch.zeros_like(coeffs))
