"""Interface to Wannier90 (mirror of src/external/wannier_shared.jl and ext/DFTKWannier90Ext.jl).

An SCF result is unfolded to the full Monkhorst-Pack grid (unfold_bz) and written as the Wannier90 input files: `.win`,
`.eig`, `.amn` (projections A_k), `.mmn` (overlaps M^{k,b} with every neighbour k+b of the `.nnkp` list) and, for plotting,
the formatted `UNK` files.  The matrices of all k-points are one batched device product each (dftk_b200_overlap_multi): the
neighbour of a k-point is addressed through an index table built on the device (dftk_b200_remap_tables with M = I and
delta = G_shift), so no gathered copy of ψ_{k+b} is formed.  Projections are evaluated on the device: the phase
exp(-2πi (k+G)·c) by dftk_b200_build_projectors with the centre as the atom, the hydrogenic radial part by
dftk_b200_radial_transform.  Indices are 0-based here; the files are 1-based, as Wannier90 reads them."""
import math
import os
import shutil
import subprocess
from datetime import datetime
from typing import NamedTuple

import numpy as np
import torch

from ._lib import check, c_vp
from .basis import MonkhorstPack
from .device import _ptr
from .pseudo import solid_harmonic_real
from .transfer import remap_tables, _lookup, _single_rank, unfold_bz

HARTREE_IN_EV = 27.211386245988     # CODATA 2018
_I3 = np.eye(3, dtype=np.int32)


# ------------------------------------------------------------------ device product
def overlap_multi(ctx, n_a, n_b, pairs):
    """dftk_b200_overlap_multi, one call for all pairs (A, B, idx, n_G): C_p[m, n] = Σ_{j < n_G} conj(A[m, j]) B[n, idx[j]]
    (idx None: j itself; -1: nothing) for the first n_a rows of A and n_b rows of B.  Returns (n_pairs, n_a, n_b) on the
    device.  Consecutive pairs with the same A read it once."""
    n = len(pairs)
    C = torch.empty((n, n_b, n_a), dtype=torch.complex128, device=ctx.device)     # column-major n_a x n_b per pair
    if n == 0:
        return C.transpose(1, 2)
    for A, B, idx, n_G in pairs:
        assert A.is_contiguous() and B.is_contiguous() and A.dtype == B.dtype == torch.complex128
        assert A.shape[0] >= n_a and B.shape[0] >= n_b and n_G <= A.shape[1]
        assert idx is None or (idx.is_contiguous() and idx.dtype == torch.int64 and idx.numel() == n_G)
    P = c_vp * n
    arr = lambda vals: np.ascontiguousarray(vals, dtype=np.int64)
    ld_a, ld_b, n_G = arr([p[0].shape[1] for p in pairs]), arr([p[1].shape[1] for p in pairs]), arr([p[3] for p in pairs])
    idx = P(*[None if p[2] is None else p[2].data_ptr() for p in pairs]) if any(p[2] is not None for p in pairs) else None
    check(ctx.L.dftk_b200_overlap_multi(ctx.h, n, n_a, n_b, P(*[p[0].data_ptr() for p in pairs]), _ptr(ld_a), _ptr(n_G),
                                        P(*[p[1].data_ptr() for p in pairs]), _ptr(ld_b), idx, _ptr(C)), ctx.h)
    return C.transpose(1, 2)


# ------------------------------------------------------------------ projections (wannier_shared.jl:6-71)
def _p_cart(basis, ps):
    return ps @ basis._recip.T


def _with_phase(basis, ps, center, ff):
    """exp(-2πi p·center) ff on the device (the projector-table builder with the centre as the only atom)."""
    ctx = basis.architecture.ctx
    n = ps.shape[0]
    out = torch.empty((1, n), dtype=torch.complex128, device=ps.device)
    if n == 0:
        return out[0]
    pos = np.ascontiguousarray(np.asarray(center, dtype=np.float64).reshape(3))
    ff = ff.to(torch.complex128).reshape(1, n).contiguous()
    check(ctx.L.dftk_b200_build_projectors(ctx.h, n, _ptr(ps.T.contiguous()), 1, _ptr(pos), 1, _ptr(ff), _ptr(out)), ctx.h)
    return out[0]


class GaussianWannierProjection:
    """A Gaussian-shaped initial guess (an s- or σ-like orbital) centred at `center` (reduced coordinates):
    exp(2π(-i p·c - |p_cart|²/4))."""

    def __init__(self, center):
        self.center = np.asarray(center, dtype=float)

    def __call__(self, basis, ps):
        pc = _p_cart(basis, ps)
        return _with_phase(basis, ps, self.center, torch.exp(-(math.pi / 2) * (pc * pc).sum(dim=1)))


def radial_hydrogenic(r, n, alpha=1.0):
    """src/common/hydrogenic.jl: the radial functions of the Wannier90 user guide, table 3.3 (n = 1, 2, 3)."""
    r = np.asarray(r, dtype=float)
    if n == 1:
        return 2 * alpha ** 1.5 * np.exp(-alpha * r)
    if n == 2:
        return 2 ** -1.5 * alpha ** 1.5 * (2 - alpha * r) * np.exp(-alpha * r / 2)
    if n == 3:
        return math.sqrt(4 / 27) * alpha ** 1.5 * (1 - 2 / 3 * alpha * r + 2 / 27 * alpha ** 2 * r ** 2) * np.exp(-alpha * r / 3)
    raise ValueError(f"n = {n} is not supported")


def hydrogenic_mesh(alpha):
    """The logarithmic mesh of pw2wannier90 (wannier_shared.jl:40-49): x = -6 : 0.025 : log(10), r = exp(x)/α, dr = r dx."""
    xmin, dx, rmax = -6.0, 0.025, 10.0
    n_r = int(round((math.log(rmax) - xmin) / dx)) + 1
    r = np.exp(xmin + dx * np.arange(n_r)) / alpha
    return r, r * dx


class HydrogenicWannierProjection:
    """A hydrogenic initial guess with quantum numbers (n, l, m) centred at `center` (reduced coordinates); `alpha` is the
    diffusivity Z/a.  The value is the reference's (-i)^l ylm_real(p̂) Σ r² R dr j_l(|p| r) exp(-2πi p·c) times 4π, which
    compute_amn_kpoint normalises away.  l <= 3."""

    def __init__(self, center, n, l, m, alpha):
        if not (0 <= l <= 3 and -l <= m <= l):
            raise ValueError("HydrogenicWannierProjection needs 0 <= l <= 3 and |m| <= l")
        self.center, self.n, self.l, self.m, self.alpha = np.asarray(center, dtype=float), int(n), int(l), int(m), float(alpha)

    def __call__(self, basis, ps):
        ctx = basis.architecture.ctx
        pc = _p_cart(basis, ps)
        q = torch.linalg.norm(pc, dim=1).contiguous()
        r, dr = hydrogenic_mesh(self.alpha)
        g = np.ascontiguousarray((r ** 2 * radial_hydrogenic(r, self.n, self.alpha) * dr).reshape(1, -1))
        r_d, g_d = torch.from_numpy(r).to(ps.device), torch.from_numpy(g).to(ps.device)
        ls = np.array([self.l], dtype=np.int32)
        F = torch.empty((1, q.numel()), dtype=torch.float64, device=ps.device)
        check(ctx.L.dftk_b200_radial_transform(ctx.h, len(r), _ptr(r_d), 1, _ptr(g_d), _ptr(ls), q.numel(), _ptr(q), _ptr(F)),
              ctx.h)
        # F = 4π/|p|^l Σ g j_l(|p| r) and the solid harmonic carries |p|^l: together 4π ylm_real(p̂) Σ g j_l
        ff = F[0] * solid_harmonic_real(self.l, self.m, pc) * (-1j) ** self.l
        return _with_phase(basis, ps, self.center, ff)


def default_wannier_centers(n_wannier, generator=None):
    """Random Gaussian guesses in reduced coordinates (the reference's default for run_wannier90)."""
    rng = generator if generator is not None else np.random.default_rng()
    return [GaussianWannierProjection(rng.random(3)) for _ in range(n_wannier)]


# ------------------------------------------------------------------ matrices
def _projection_table(basis, kpt, projections):
    """(n_wannier, n_G) table of the l²-normalised projections at the k+G of kpt (compute_amn_kpoint's coeffs_gn_per)."""
    ps = basis.Gplusk_vectors(kpt).contiguous()
    rows = []
    for proj in projections:
        g = torch.as_tensor(proj(basis, ps), device=ps.device).to(torch.complex128).reshape(-1)
        rows.append(g / torch.linalg.norm(g))
    return torch.stack(rows).contiguous()


def _check_bands(ψk, n_bands):
    if ψk.shape[0] < n_bands:
        raise ValueError(f"n_bands = {n_bands} exceeds the {ψk.shape[0]} bands of ψ")


def _amn_all(basis, ψ, projections, n_bands):
    """A_k of every k-block, one device call: (n_k, n_bands, n_wannier) on the host."""
    tables = [_projection_table(basis, kpt, projections) for kpt in basis.kpoints]
    pairs = []
    for ψk, kpt, g in zip(ψ, basis.kpoints, tables):
        _check_bands(ψk, n_bands)
        pairs.append((ψk.to(torch.complex128).contiguous(), g, None, kpt.n_G))
    return overlap_multi(basis.architecture.ctx, n_bands, len(projections), pairs).cpu().numpy()


def compute_amn_kpoint(basis, kpt, ψk, projections, n_bands):
    """wannier_shared.jl:278-298: [A_k]_{mn} = <ψ_m^k | g_n^per> with each g_n l²-normalised on the k+G sphere."""
    _check_bands(ψk, n_bands)
    g = _projection_table(basis, kpt, projections)
    return overlap_multi(basis.architecture.ctx, n_bands, len(projections),
                         [(ψk.to(torch.complex128).contiguous(), g, None, kpt.n_G)])[0].cpu().numpy()


def _mmn_pairs(basis, ψ, nnkpts, n_bands):
    ctx = basis.architecture.ctx
    blocks = [p.to(torch.complex128).contiguous() for p in ψ]
    pairs = []
    for ik, ikb, G_shift in nnkpts:
        k, kb = basis.kpoints[ik], basis.kpoints[ikb]
        _check_bands(blocks[ik], n_bands)
        _check_bands(blocks[ikb], n_bands)
        idx, _ = remap_tables(ctx, k.G_vectors, _I3, np.asarray(G_shift), _lookup(basis, kb), basis.fft_size)
        pairs.append((blocks[ik], blocks[ikb], idx, k.n_G))
    return pairs


def _identity_if_zero(M):
    """The reference's `iszero(Mkb) && return I`."""
    if not M.any():
        return np.eye(M.shape[0], dtype=M.dtype)
    return M


def _mmn_all(basis, ψ, nnkpts, n_bands):
    """M^{k,b} of every (ik, ik_plus_b, G_shift) of the list, one device call: (n_pairs, n_bands, n_bands) on the host."""
    M = overlap_multi(basis.architecture.ctx, n_bands, n_bands, _mmn_pairs(basis, ψ, nnkpts, n_bands)).cpu().numpy()
    return np.stack([_identity_if_zero(m) for m in M]) if len(M) else M


def overlap_Mmn_k_kpb(basis, ψ, ik, ik_plus_b, G_shift, n_bands):
    """wannier_shared.jl:220-241: [M^{k,b}]_{mn} = <u_{m,k} | u_{n,k+b}>, with u_{n,k+G_shift} = e^{-i G_shift·r} u_{n,k}
    taking care of a neighbour in another cell.  ik, ik_plus_b 0-based; the identity when every overlap vanishes."""
    return _mmn_all(basis, ψ, [(ik, ik_plus_b, G_shift)], n_bands)[0]


# ------------------------------------------------------------------ files
class NnkPt(NamedTuple):
    ik: int                 # 0-based
    ik_plus_b: int          # 0-based
    G_shift: tuple


class Nnkp(NamedTuple):
    nntot: int
    nnkpts: list


def _now():
    return datetime.now().isoformat(timespec="milliseconds")


def _w90_value(v):
    if isinstance(v, (bool, np.bool_)):
        return "true" if v else "false"
    return str(v)


def write_w90_win(fileprefix, basis, *, bands_plot=False, wannier_plot=False, **kwargs):
    """wannier_shared.jl:73-134: the .win input file; Wannier90 parameters are passed as keywords (num_bands and num_wann
    are required)."""
    if "num_bands" not in kwargs or "num_wann" not in kwargs:
        raise ValueError("write_w90_win needs num_bands and num_wann")
    if not isinstance(basis.kgrid, MonkhorstPack):
        raise ValueError("The basis must be constructed from a MP grid.")
    if bands_plot:
        raise NotImplementedError("bands_plot needs a high-symmetry k-path (irrfbz_path), which is not available")
    model = basis.model
    with open(fileprefix + ".win", "w") as fp:
        fp.write(f"! Generated by DFTK.jl at {_now()}\n\n")
        for key, value in kwargs.items():
            fp.write("%-20s =   %-30s\n" % (key, _w90_value(value)))
        if wannier_plot:
            fp.write("wvfn_formatted = True\n")
            fp.write("wannier_plot   = True\n")
        fp.write("\n" + "!" * 20 + " System \n\n\n")
        fp.write("begin unit_cell_cart\nbohr\n")
        for vec in np.asarray(model.lattice).T:              # lattice vectors are rows in Wannier90
            fp.write("%10.6f %10.6f %10.6f \n" % tuple(vec))
        fp.write("end unit_cell_cart \n\n")
        fp.write("begin atoms_frac\n")
        for atom, pos in zip(model.atoms, model.positions):
            fp.write("%-2s %10.6f %10.6f %10.6f \n" % ((atom.symbol,) + tuple(np.asarray(pos, dtype=float))))
        fp.write("end atoms_frac\n\n")
        fp.write("!" * 20 + " k_points\n\n")
        size = basis.kgrid.kgrid_size
        fp.write(f"mp_grid : {size[0]} {size[1]} {size[2]}\n\n")
        fp.write("begin kpoints\n")
        for kpt in basis.kpoints:
            fp.write("%10.10f %10.10f %10.10f\n" % tuple(kpt.coordinate))
        fp.write("end kpoints\n")


def read_w90_nnkp(fileprefix):
    """wannier_shared.jl:137-176: (nntot, nnkpts) of the .nnkp file written by `wannier90.x -pp`; each entry is
    (ik, ik_plus_b, G_shift) with 0-based k-point indices."""
    fn = fileprefix + ".nnkp"
    if not os.path.isfile(fn):
        raise FileNotFoundError(f"Expected file {fn} not found.")
    with open(fn) as fh:
        lines = fh.read().splitlines()
    ib, ie = lines.index("begin nnkpts"), lines.index("end nnkpts")
    nntot = int(lines[ib + 1])
    nnkpts = []
    for line in lines[ib + 2:ie]:
        v = [int(s) for s in line.split()]
        if len(v) != 5:
            raise ValueError(f"malformed nnkpts line: {line!r}")
        nnkpts.append(NnkPt(v[0] - 1, v[1] - 1, tuple(v[2:5])))
    return Nnkp(nntot, nnkpts)


def write_w90_eig(fileprefix, eigenvalues, *, n_bands):
    """wannier_shared.jl:179-191: the eigenvalues in eV."""
    with open(fileprefix + ".eig", "w") as fp:
        for k, εk in enumerate(eigenvalues, start=1):
            for n, ε in enumerate(np.asarray(εk)[:n_bands], start=1):
                fp.write("%3i  %3i   %25.18f \n" % (n, k, float(ε) * HARTREE_IN_EV))


def _krange_spin(basis, spin):
    return [ik for ik, kpt in enumerate(basis.kpoints) if kpt.spin == spin - 1]


def write_w90_unk(fileprefix, basis, ψ, *, n_bands, spin=1):
    """wannier_shared.jl:194-212: the formatted UNK%05i.%i files of the real-space periodic parts u_nk (ifft(basis, kpt, ψ)
    normalisation, 1/√Ω), x fastest."""
    nx, ny, nz = basis.fft_size
    for ik in _krange_spin(basis, spin):
        kpt = basis.kpoints[ik]
        _check_bands(ψ[ik], n_bands)
        cube = torch.zeros((n_bands, basis.N), dtype=torch.complex128, device=kpt.mapping.device)
        cube[:, kpt.mapping] = ψ[ik][:n_bands].to(torch.complex128)
        u = basis.ifft(cube).cpu().numpy()
        with open(os.path.join(os.path.dirname(fileprefix), "UNK%05i.%i" % (ik + 1, spin)), "w") as fp:
            fp.write(f"{nx} {ny} {nz} {ik + 1} {n_bands}\n")
            for row in u:
                np.savetxt(fp, np.column_stack([row.real, row.imag]), fmt="%25.18f %25.18f")


def write_w90_mmn(fileprefix, basis, ψ, nnkp, *, n_bands):
    """wannier_shared.jl:243-256: the overlaps of every pair of the nnkp list (one device call), column-major."""
    M = _mmn_all(basis, ψ, nnkp.nnkpts, n_bands)
    with open(fileprefix + ".mmn", "w") as fp:
        fp.write(f"Generated by DFTK at {_now()}\n")
        fp.write(f"{n_bands}  {len(ψ)}  {nnkp.nntot}\n")
        for (ik, ikb, G_shift), m in zip(nnkp.nnkpts, M):
            fp.write("%i  %i  %i  %i  %i \n" % ((ik + 1, ikb + 1) + tuple(int(g) for g in G_shift)))
            for v in m.T.reshape(-1):
                fp.write("%22.18f %22.18f \n" % (v.real, v.imag))


def write_w90_amn(fileprefix, basis, projections, ψ, *, n_bands):
    """wannier_shared.jl:301-322: A_k of every k-point (one device call), column-major."""
    A = _amn_all(basis, ψ, projections, n_bands)
    with open(fileprefix + ".amn", "w") as fp:
        fp.write(f"Generated by DFTK at {_now()}\n")
        fp.write(f"{n_bands}   {len(basis.kpoints)}  {len(projections)}\n")
        for ik, Ak in enumerate(A, start=1):
            for n in range(Ak.shape[1]):
                for m in range(Ak.shape[0]):
                    v = Ak[m, n]
                    fp.write("%3i %3i %3i  %22.18f %22.18f \n" % (m + 1, n + 1, ik, v.real, v.imag))


# ------------------------------------------------------------------ drivers
def _check_supported(scfres, kwargs):
    basis = scfres["basis"]
    if basis.model.spin_polarization not in ("none", "spinless"):
        raise NotImplementedError("Wannierisation supports spin_polarization none or spinless only")
    _single_rank(basis, "write_wannier90_files")
    if kwargs.get("bands_plot"):
        raise NotImplementedError("bands_plot needs a high-symmetry k-path (irrfbz_path), which is not available")


def write_wannier90_files(preprocess_call, scfres, *, n_bands, n_wannier, projections, fileprefix, wannier_plot, **kwargs):
    """wannier_shared.jl:333-368: unfold the result to the full k-grid, write the .win file, call `preprocess_call()` (which
    must return the read_w90_nnkp result), then write .eig, .amn, .mmn and, with wannier_plot, the UNK files."""
    _check_supported(scfres, kwargs)
    if len(projections) != n_wannier:
        raise ValueError("need one projection per Wannier function")
    su = unfold_bz(scfres)
    basis, ψ = su["basis"], su["psi"]
    d = os.path.dirname(fileprefix)
    if d:
        os.makedirs(d, exist_ok=True)
    write_w90_win(fileprefix, basis, num_wann=n_wannier, num_bands=n_bands, wannier_plot=wannier_plot, **kwargs)
    nnkp = preprocess_call()
    write_w90_eig(fileprefix, su["eigenvalues"], n_bands=n_bands)
    write_w90_amn(fileprefix, basis, projections, ψ, n_bands=n_bands)
    write_w90_mmn(fileprefix, basis, ψ, nnkp, n_bands=n_bands)
    if wannier_plot:
        write_w90_unk(fileprefix, basis, ψ, n_bands=n_bands, spin=1)


def wannier90_executable():
    """`$WANNIER90` when set, else `wannier90.x` from PATH."""
    exe = os.environ.get("WANNIER90") or shutil.which("wannier90.x")
    if not exe or not os.path.isfile(exe):
        raise FileNotFoundError("wannier90.x not found: put it on PATH or set WANNIER90 to its path")
    return exe


def run_wannier90(scfres, *, n_bands=None, n_wannier=None, projections=None, fileprefix=os.path.join("wannier90", "wannier"),
                  wannier_plot=False, **kwargs):
    """ext/DFTKWannier90Ext.jl: write the input files, run `wannier90.x -pp <prefix>` and `wannier90.x <prefix>` in the
    prefix's directory.  Defaults as in the reference: n_bands = scfres["n_bands_converge"], n_wannier = n_bands, random
    Gaussian centres.  Returns fileprefix."""
    _check_supported(scfres, kwargs)
    exe = wannier90_executable()
    n_bands = scfres["n_bands_converge"] if n_bands is None else n_bands
    n_wannier = n_bands if n_wannier is None else n_wannier
    projections = default_wannier_centers(n_wannier) if projections is None else projections
    prefix, d = os.path.basename(fileprefix), os.path.dirname(fileprefix) or "."

    def preprocess():
        subprocess.run([exe, "-pp", prefix], cwd=d, check=True)
        return read_w90_nnkp(fileprefix)

    write_wannier90_files(preprocess, scfres, n_bands=n_bands, n_wannier=n_wannier, projections=projections,
                          fileprefix=fileprefix, wannier_plot=wannier_plot, **kwargs)
    subprocess.run([exe, prefix], cwd=d, check=True)
    return fileprefix
