"""Moving SCF results between bases (mirror of src/transfer.jl:10-178, src/interpolation.jl:9-89, src/supercell.jl and
apply_symop / unfold_bz of src/symmetry.jl:229-270,459-531).

Orbitals stay on the device as (n_bands, n_G) complex128 blocks and densities as (n_spin, N) cubes.  Every orbital move is
one batched sphere remap of libdftk_b200 (dftk_b200_sphere_remap) over index/phase tables the library builds on the
device (dftk_b200_remap_tables); densities move by the Fourier block copy (transfer_density) or the periodic quadratic
B-spline (interpolate_density) between the library's own cube FFTs.  Indices are 0-based (Julia: 1-based)."""
import math
import warnings

import numpy as np
import torch

from ._lib import check, c_vp
from .basis import PlaneWaveBasis, MonkhorstPack, Kpoint, normalize_kpoint_coordinate
from .device import FFTGrid, _ptr
from .model import Model, SYMMETRY_TOLERANCE

_I3 = np.eye(3, dtype=np.int32)


# ------------------------------------------------------------------ device primitives
def _lookup(basis, kpt):
    """Cube index -> row of `kpt`'s sphere, -1 outside it (int64, device); cached on the k-point."""
    lk = getattr(kpt, "_cube_lookup", None)
    if lk is None or lk.numel() != basis.N:
        lk = torch.full((basis.N,), -1, dtype=torch.int64, device=kpt.mapping.device)
        lk[kpt.mapping] = torch.arange(kpt.n_G, dtype=torch.int64, device=kpt.mapping.device)
        kpt._cube_lookup = lk
    return lk


def remap_tables(ctx, G, M, delta, lookup, fft_size, tau=None):
    """dftk_b200_remap_tables: for the destination G vectors G (n, 3) int64 (device), idx[j] = lookup[M (G_j + delta)]
    (-1 outside the source cube or sphere) and, when `tau` is given, phase[j] = exp(-2πi (G_j + delta)·tau)."""
    G = G.contiguous()
    n = G.shape[0]
    idx = torch.empty(n, dtype=torch.int64, device=G.device)
    phase = None if tau is None else torch.empty(n, dtype=torch.complex128, device=G.device)
    Mh = np.ascontiguousarray(np.rint(M), dtype=np.int32)
    dh = np.ascontiguousarray(np.rint(delta), dtype=np.int32)
    th = None if tau is None else np.ascontiguousarray(tau, dtype=np.float64)
    nx, ny, nz = (int(v) for v in fft_size)
    check(ctx.L.dftk_b200_remap_tables(ctx.h, n, _ptr(G), _ptr(Mh), _ptr(dh), _ptr(th), _ptr(lookup.contiguous()),
                                       nx, ny, nz, _ptr(idx), _ptr(phase)), ctx.h)
    return idx, phase


def sphere_remap(ctx, pairs):
    """dftk_b200_sphere_remap, one launch: for each (src, dst, idx, phase, row_offset),
    dst[row_offset + b, j] = phase[j] src[b, idx[j]] (idx -1 -> 0, phase None -> 1) for every row b of src."""
    n = len(pairs)
    if n == 0:
        return
    for src, dst, idx, _, off in pairs:
        assert src.is_contiguous() and dst.is_contiguous() and idx.is_contiguous()
        assert src.dtype == dst.dtype == torch.complex128 and idx.numel() == dst.shape[1]
        assert off + src.shape[0] <= dst.shape[0] and dst.data_ptr() != src.data_ptr()
    P = c_vp * n
    arr = lambda vals: np.ascontiguousarray(vals, dtype=np.int64)
    ld_src, ld_dst = arr([p[0].shape[1] for p in pairs]), arr([p[1].shape[1] for p in pairs])
    offs, nbs, n_dst = arr([p[4] for p in pairs]), arr([p[0].shape[0] for p in pairs]), arr([p[2].numel() for p in pairs])
    ph = P(*[None if p[3] is None else p[3].data_ptr() for p in pairs]) if any(p[3] is not None for p in pairs) else None
    check(ctx.L.dftk_b200_sphere_remap(ctx.h, n, P(*[p[0].data_ptr() for p in pairs]), _ptr(ld_src),
                                       P(*[p[1].data_ptr() for p in pairs]), _ptr(ld_dst), _ptr(offs), _ptr(nbs),
                                       P(*[p[2].data_ptr() for p in pairs]), _ptr(n_dst), ph), ctx.h)


def _delta_G(k_in, k_out):
    dG = np.asarray(k_out, dtype=float) - np.asarray(k_in, dtype=float)
    if np.max(np.abs(dG - np.round(dG))) > SYMMETRY_TOLERANCE:
        raise ValueError("kpt_out must equal kpt_in + ΔG for an integer ΔG")
    return np.round(dG).astype(np.int64)


def _check_lattices(basis_in, basis_out):
    if not np.array_equal(basis_in.model.lattice, basis_out.model.lattice):
        raise ValueError("both bases need the same lattice")


# ------------------------------------------------------------------ transfer.jl
def _axis_blocks(n_in, n_out):
    if n_in <= n_out:
        a, b = -(-n_in // 2), n_in // 2
        return (slice(0, a), slice(a, n_in)), (slice(0, a), slice(n_out - b, n_out))
    a, b = -(-n_out // 2), n_out // 2
    return (slice(0, a), slice(n_in - b, n_in)), (slice(0, a), slice(a, n_out))


def transfer_mapping(basis_in, *args):
    """transfer.jl:10-83.  transfer_mapping(basis_in, basis_out): the 8 pairs (block_in, block_out) of per-axis (x, y, z)
    slices with x_out[block_out] = x_in[block_in] transferring Fourier cubes.  transfer_mapping(basis_in, kpt_in,
    basis_out, kpt_out): index tensors (idcs_in, idcs_out) with ψk_out[idcs_out] = ψk_in[idcs_in]; kpt_out may be
    kpt_in + ΔG."""
    if len(args) == 1:
        basis_out = args[0]
        _check_lattices(basis_in, basis_out)
        ax = [_axis_blocks(a, b) for a, b in zip(basis_in.fft_size, basis_out.fft_size)]
        return [((ax[0][0][i], ax[1][0][j], ax[2][0][k]), (ax[0][1][i], ax[1][1][j], ax[2][1][k]))
                for k in range(2) for j in range(2) for i in range(2)]
    kpt_in, basis_out, kpt_out = args
    _check_lattices(basis_in, basis_out)
    dG = _delta_G(kpt_in.coordinate, kpt_out.coordinate)
    idcs_in = torch.arange(kpt_in.n_G, device=kpt_in.mapping.device)
    if kpt_in is kpt_out:
        return idcs_in, idcs_in
    # position of every input row in kpt_out's sphere: G_in - ΔG looked up on basis_out's cube
    pos, _ = remap_tables(basis_out.architecture.ctx, kpt_in.G_vectors, _I3, -dG, _lookup(basis_out, kpt_out),
                          basis_out.fft_size)
    keep = pos >= 0
    return idcs_in[keep], pos[keep]


def _transfer_pair(ψk, basis_in, kpt_in, basis_out, kpt_out):
    dG = _delta_G(kpt_in.coordinate, kpt_out.coordinate)
    if ψk.shape[-1] != kpt_in.n_G:
        raise ValueError("ψk does not match the G vectors of kpt_in")
    idx, _ = remap_tables(basis_in.architecture.ctx, kpt_out.G_vectors, _I3, dG, _lookup(basis_in, kpt_in),
                          basis_in.fft_size)
    src = ψk.to(torch.complex128).contiguous()
    dst = torch.empty((src.shape[0], kpt_out.n_G), dtype=torch.complex128, device=src.device)
    return (src, dst, idx, None, 0)


def transfer_blochwave_kpt(ψk, basis_in, kpt_in, basis_out, kpt_out):
    """transfer.jl:112-124: ψk (n_bands, n_G(kpt_in)) on kpt_out; coefficients outside either sphere are dropped."""
    if kpt_in is kpt_out:
        return ψk.clone()
    _check_lattices(basis_in, basis_out)
    pair = _transfer_pair(ψk, basis_in, kpt_in, basis_out, kpt_out)
    sphere_remap(basis_in.architecture.ctx, [pair])
    return pair[1]


def transfer_blochwave(ψ, basis_in, basis_out):
    """transfer.jl:129-150: all k-blocks of this rank in one remap launch."""
    _check_lattices(basis_in, basis_out)
    if len(ψ) != len(basis_in.kpoints) or len(basis_in.kpoints) != len(basis_out.kpoints):
        raise ValueError("ψ, basis_in and basis_out need the same k-blocks")
    if list(basis_in.krange_thisproc_allspin) != list(basis_out.krange_thisproc_allspin):
        raise NotImplementedError("transfer_blochwave between bases whose k-blocks are laid out differently over the ranks")
    for ki, ko in zip(basis_in.kpoints, basis_out.kpoints):
        if not np.array_equal(ki.coordinate, ko.coordinate) or ki.spin != ko.spin:
            raise ValueError("basis_in and basis_out need the same k-points")
    pairs = [_transfer_pair(ψk, basis_in, ki, basis_out, ko) for ψk, ki, ko in zip(ψ, basis_in.kpoints, basis_out.kpoints)]
    sphere_remap(basis_in.architecture.ctx, pairs)
    return [p[1] for p in pairs]


def transfer_density(ρ, basis_in, basis_out):
    """transfer.jl:165-178: the Fourier coefficients of ρ (n_spin, N_in) kept where both cubes hold them.  For an
    even-sized small grid small -> big -> small is not the identity (its unmatched component has no partner)."""
    _check_lattices(basis_in, basis_out)
    ctx = basis_in.architecture.ctx
    f = basis_in.fft(ρ.reshape(-1, basis_in.N)).contiguous()
    out = torch.empty((f.shape[0], basis_out.N), dtype=torch.complex128, device=f.device)
    check(ctx.L.dftk_b200_fourier_block_copy(ctx.h, _ptr(f), *basis_in.fft_size, _ptr(out), *basis_out.fft_size,
                                             f.shape[0]), ctx.h)
    return basis_out.irfft(out)


# ------------------------------------------------------------------ interpolation.jl
_GRIDS = {}


def _unit_grid(ctx, size):
    key = (id(ctx), tuple(size))
    if key not in _GRIDS:
        _GRIDS[key] = FFTGrid(ctx, size, 1.0)
    return _GRIDS[key]


def _ctx_of(t):
    from .architecture import B200
    return B200(device=t.device.index if t.device.index is not None else torch.cuda.current_device()).ctx


def _bspline(ρ, grid_in, grid_out, rep, ctx):
    """ρ (n_spin, N_in) -> (n_spin, N_out) on the device; see interpolate_density."""
    ρ = ρ.to(torch.float64).contiguous()
    n_spin = ρ.shape[0]
    out = torch.empty((n_spin, int(np.prod(grid_out))), dtype=torch.float64, device=ρ.device)
    r = np.ascontiguousarray(rep, dtype=np.int32)
    direct = all(a * b == c for a, b, c in zip(grid_in, rep, grid_out))
    if direct:
        coef = ρ
    else:
        grid = _unit_grid(ctx, grid_in)
        c = ρ.to(torch.complex128).contiguous()
        grid.fft_cube(c, -1)
        check(ctx.L.dftk_b200_bspline2_prefilter(ctx.h, _ptr(c), *grid_in, n_spin), ctx.h)
        grid.fft_cube(c, +1)
        coef = (c.real / grid.N).contiguous()
    check(ctx.L.dftk_b200_bspline2_evaluate(ctx.h, _ptr(coef), *grid_in, _ptr(r), _ptr(out), *grid_out, n_spin,
                                            int(direct)), ctx.h)
    return out


def _as_cubes(ρ, grid):
    """(n_spin, N) or (n_spin, nz, ny, nx) -> (n_spin, N)."""
    return ρ.reshape(ρ.shape[0], int(np.prod(grid)))


def supercell_size(lattice_in, lattice_out):
    """interpolation.jl:41-53: the integer repetition of each lattice vector, with the reference's warning."""
    lattice_in, lattice_out = np.asarray(lattice_in, dtype=float), np.asarray(lattice_out, dtype=float)
    zin, zout = ~lattice_in.any(axis=0), ~lattice_out.any(axis=0)
    if not np.array_equal(zin, zout):
        raise ValueError("the two lattices need the same dimension")
    rep = [1 if zin[i] else int(round(np.linalg.norm(lattice_out[:, i]) / np.linalg.norm(lattice_in[:, i])))
           for i in range(3)]
    for i in range(3):
        if np.linalg.norm(rep[i] * lattice_in[:, i] - lattice_out[:, i]) > 0.3 * np.linalg.norm(lattice_out[:, i]):
            warnings.warn(f"In direction {i + 1}, the output lattice is very different from the input lattice")
    return rep


def interpolate_density(ρ, *args):
    """interpolation.jl:9-89, periodic quadratic B-spline (Interpolations.jl BSpline(Quadratic(Periodic(OnCell())))):
      interpolate_density(ρ, basis_in, basis_out)      ρ (n_spin, N_in) -> (n_spin, N_out); a supercell when the lattices differ
      interpolate_density(ρ, grid_out)                 ρ (n_spin, nz, ny, nx) -> (n_spin, nz', ny', nx')
      interpolate_density(ρ, grid_in, grid_out, lattice_in, lattice_out)   ρ (n_spin, N_in) or 4-D as above
    Grid sizes are (nx, ny, nz) like fft_size.  Output point (i/nx', j/ny', k/nz') of the output cell is evaluated on the
    input grid's periodic spline; for a supercell the tiling is folded into the index arithmetic.  Equal grids (and an output
    grid that is exactly the tiled input grid) give a copy, as in the reference."""
    if len(args) == 2 and isinstance(args[0], PlaneWaveBasis):
        basis_in, basis_out = args
        if basis_in.model.n_spin_components != ρ.shape[0]:
            raise ValueError("ρ does not match basis_in")
        if np.array_equal(basis_in.model.lattice, basis_out.model.lattice):
            rep = [1, 1, 1]
        else:
            rep = supercell_size(basis_in.model.lattice, basis_out.model.lattice)
        return _bspline(_as_cubes(ρ, basis_in.fft_size), basis_in.fft_size, basis_out.fft_size, rep,
                        basis_in.architecture.ctx)
    if len(args) == 1:
        if ρ.dim() != 4:
            raise ValueError("interpolate_density(ρ, grid_out) needs ρ of shape (n_spin, nz, ny, nx)")
        grid_in = (ρ.shape[3], ρ.shape[2], ρ.shape[1])
        grid_out = tuple(int(v) for v in args[0])
        out = _bspline(_as_cubes(ρ, grid_in), grid_in, grid_out, [1, 1, 1], _ctx_of(ρ))
        return out.reshape(ρ.shape[0], grid_out[2], grid_out[1], grid_out[0])
    if len(args) == 4:
        grid_in, grid_out = tuple(int(v) for v in args[0]), tuple(int(v) for v in args[1])
        rep = supercell_size(args[2], args[3])
        out = _bspline(_as_cubes(ρ, grid_in), grid_in, grid_out, rep, _ctx_of(ρ))
        return out if ρ.dim() == 2 else out.reshape(ρ.shape[0], grid_out[2], grid_out[1], grid_out[0])
    raise TypeError("interpolate_density(ρ, basis_in, basis_out), (ρ, grid_out) or (ρ, grid_in, grid_out, lattice_in, "
                    "lattice_out)")


# ------------------------------------------------------------------ symmetry.jl
def _invS(symop):
    return np.rint(np.linalg.inv(symop.S)).astype(np.int32)


def _symop_kshift(symop, kcoord):
    Sk_raw = symop.S @ np.asarray(kcoord, dtype=float)
    Sk = normalize_kpoint_coordinate(Sk_raw)
    return Sk, np.rint(Sk - Sk_raw).astype(np.int64)


def _symop_pair(symop, basis, kpoint, ψk, Skpoint, kshift):
    idx, phase = remap_tables(basis.architecture.ctx, Skpoint.G_vectors, _invS(symop), kshift, _lookup(basis, kpoint),
                              basis.fft_size, tau=symop.tau)
    src = ψk.to(torch.complex128).contiguous()
    dst = torch.empty((src.shape[0], Skpoint.n_G), dtype=torch.complex128, device=src.device)
    return (src, dst, idx, phase, 0)


def apply_symop(symop, basis, kpoint, ψk):
    """symmetry.jl:229-270: (Skpoint, ψSk) with u_Sk(G) = exp(-2πi G·τ) u_k(S⁻¹G), G running over the sphere of
    Sk reduced to [-1/2, 1/2) (G + kshift in the formula)."""
    if symop.isone():
        return kpoint, ψk
    k = np.asarray(kpoint.coordinate, dtype=float)
    if not np.all((-0.5 <= k) & (k < 0.5)):
        raise ValueError("kpoint coordinate must lie in [-1/2, 1/2)")
    Sk, kshift = _symop_kshift(symop, k)
    Skpoint = None
    for kp in basis.kpoints:
        d = kp.coordinate - Sk
        if np.all(np.abs(d - np.round(d)) < SYMMETRY_TOLERANCE) and kp.spin == kpoint.spin:
            Skpoint = kp
            break
    if Skpoint is None:
        mapping = torch.nonzero(basis.sphere_mask(Sk)).reshape(-1)
        Skpoint = Kpoint(kpoint.spin, Sk, mapping, basis.G_vectors[mapping])
    pair = _symop_pair(symop, basis, kpoint, ψk, Skpoint, kshift)
    sphere_remap(basis.architecture.ctx, [pair])
    return Skpoint, pair[1]


def _single_rank(basis, what):
    if basis.comm_kpts.nranks > 1:
        raise NotImplementedError(f"{what} with k-points distributed over more than one rank")


def unfold_bz(arg):
    """symmetry.jl:459-531.  unfold_bz(basis): the same basis without k-point reduction by symmetry (it keeps the
    symmetries, used to symmetrise densities, and the FFT size).  unfold_bz(scfres): ψ carried to every k-point of the
    full grid by apply_symop (all blocks in one remap launch), eigenvalues and occupations copied, energies and `ham`
    recomputed on the unfolded basis; the total energy must be unchanged."""
    if isinstance(arg, PlaneWaveBasis):
        basis = arg
        if len(basis.symmetries) == 1:
            return basis
        _single_rank(basis, "unfold_bz")
        return PlaneWaveBasis(basis.model, Ecut=basis.Ecut, kgrid=basis.kgrid, fft_size=basis.fft_size,
                              architecture=basis.architecture, comm_kpts=basis.comm_kpts,
                              use_symmetries_for_kpoint_reduction=False,
                              _symmetries_respect_rgrid=basis.symmetries_respect_rgrid)
    scfres = arg
    basis = scfres["basis"]
    _single_rank(basis, "unfold_bz")
    bu = unfold_bz(basis)
    if bu is basis:
        return scfres
    from .hamiltonian import energy_hamiltonian
    pairs, src_of = [], []
    for ku in bu.kpoints:
        ik, op = _unfold_mapping(basis, ku)
        kshift = np.rint(ku.coordinate - op.S @ basis.kpoints[ik].coordinate).astype(np.int64)
        pairs.append(_symop_pair(op, basis, basis.kpoints[ik], scfres["psi"][ik], ku, kshift))
        src_of.append(ik)
    sphere_remap(basis.architecture.ctx, pairs)
    psi = [p[1] for p in pairs]
    eigenvalues = [np.array(scfres["eigenvalues"][ik], copy=True) for ik in src_of]
    occupation = [np.array(scfres["occupation"][ik], copy=True) for ik in src_of]
    energies, ham = energy_hamiltonian(bu, psi, occupation, rho=scfres["rho"], eigenvalues=eigenvalues, eF=scfres["eF"],
                                       hubbard_n=scfres.get("hubbard_n"))
    E0 = scfres["energies"].total
    if not abs(energies.total - E0) <= math.sqrt(np.finfo(float).eps) * max(abs(E0), abs(energies.total)):
        raise AssertionError(f"unfold_bz changed the total energy: {E0} -> {energies.total}")
    return dict(scfres, basis=bu, psi=psi, ham=ham, eigenvalues=eigenvalues, occupation=occupation,
                eigenvalues_global=eigenvalues, occupation_global=occupation)


def _unfold_mapping(basis_irred, kpt_unfolded):
    """symmetry.jl:475-487: the irreducible block and the symmetry that carries it to `kpt_unfolded`."""
    ku = normalize_kpoint_coordinate(kpt_unfolded.coordinate)
    for ik, kp in enumerate(basis_irred.kpoints):
        if kp.spin != kpt_unfolded.spin:
            continue
        for op in basis_irred.symmetries:
            if np.allclose(normalize_kpoint_coordinate(op.S @ kp.coordinate), ku, rtol=0, atol=1e-8):
                return ik, op
    raise ValueError("Invalid unfolding of BZ")


# ------------------------------------------------------------------ supercell.jl
def create_supercell(lattice, atoms, positions, supercell_size):
    """supercell.jl:5-20: lattice vectors scaled by supercell_size; for each atom its images (position + (i, j, k)) /
    supercell_size with i running fastest."""
    size = np.asarray(supercell_size, dtype=int)
    lattice_sc = np.asarray(lattice, dtype=float) * size[None, :]
    atoms_sc, positions_sc = [], []
    for atom, pos in zip(atoms, positions):
        for k in range(size[2]):
            for j in range(size[1]):
                for i in range(size[0]):
                    positions_sc.append((np.asarray(pos, dtype=float) + np.array([i, j, k])) / size)
                    atoms_sc.append(atom)
    return dict(lattice=lattice_sc, atoms=atoms_sc, positions=positions_sc)


def _no_hubbard(model):
    if "Hubbard" in model.term_names:
        raise NotImplementedError("cell_to_supercell of a model with a Hubbard term")


def _supercell_basis(basis):
    if not isinstance(basis.kgrid, MonkhorstPack):
        raise ValueError("cell_to_supercell needs a Monkhorst-Pack k-grid")
    if any(s != 0 for s in basis.kgrid.kshift):
        raise NotImplementedError("Only kshift of 0 implemented.")
    _no_hubbard(basis.model)
    model = basis.model
    size = basis.kgrid.kgrid_size
    n_cells = int(np.prod(size))
    sc = create_supercell(model.lattice, model.atoms, model.positions, size)
    moments = [m for m in model.magnetic_moments for _ in range(n_cells)]
    sc_model = Model(sc["lattice"], sc["atoms"], sc["positions"], model_name=model.model_name,
                     n_electrons=n_cells * model.n_electrons, magnetic_moments=moments, terms=model.term_types,
                     functionals=model.functionals, temperature=model.temperature, smearing=model.smearing,
                     spin_polarization=model.spin_polarization, symmetries=False)
    return PlaneWaveBasis(sc_model, Ecut=basis.Ecut, kgrid=(1, 1, 1),
                          fft_size=tuple(n * s for n, s in zip(basis.fft_size, size)),
                          architecture=basis.architecture, comm_kpts=basis.comm_kpts, _symmetries_respect_rgrid=True)


def _supercell_rows(basis, basis_supercell, kpt, Γ):
    """Supercell sphere row of every k+G row of kpt (supercell.jl:58-62, 79-82): the supercell's integer coordinates of
    k+G are diag(kgrid)·(G + k)."""
    size = torch.as_tensor(basis.kgrid.kgrid_size, dtype=torch.float64, device=kpt.G_vectors.device)
    Gs = torch.round((kpt.G_vectors.to(torch.float64) + torch.as_tensor(kpt.coordinate, device=size.device)) * size)
    cube = basis_supercell.index_G_vectors(Gs.to(torch.int64))
    rows = torch.where(cube >= 0, _lookup(basis_supercell, Γ)[cube.clamp(min=0)], torch.full_like(cube, -1))
    if bool((rows < 0).any()):
        raise ValueError("a k+G vector of the unit cell is not in the supercell's sphere")
    return rows


def cell_to_supercell(*args):
    """supercell.jl:27-129.
      cell_to_supercell(basis)                        the Γ-only basis of the supercell of the k-grid (MP grid, zero shift)
      cell_to_supercell(ψ, basis, basis_supercell)    the orbitals of an unfolded basis as one Γ block per spin channel:
                                                      columns k·n_bands + n hold ψ[k][n] (rows here: (n_k n_bands, n_G))
      cell_to_supercell(scfres)                       the whole result: unfolded, eigenvalues concatenated and sorted,
                                                      occupations at the unit cell's εF, ρ and energies on the supercell."""
    if len(args) == 3:
        ψ, basis, bs = args
        if len(basis.kgrid) != len(basis.kpoints) // basis.model.n_spin_components:
            raise ValueError("basis must be unfolded")
        out, pairs = [], []
        for Γ in bs.kpoints:
            blocks = [ik for ik, kp in enumerate(basis.kpoints) if kp.spin == Γ.spin]
            nb = ψ[blocks[0]].shape[0]
            if sum(basis.kpoints[ik].n_G for ik in blocks) != Γ.n_G:
                raise ValueError("the k+G vectors of the unit cell do not fill the supercell's sphere")
            dst = torch.empty((len(blocks) * nb, Γ.n_G), dtype=torch.complex128, device=ψ[blocks[0]].device)
            for n, ik in enumerate(blocks):
                rows = _supercell_rows(basis, bs, basis.kpoints[ik], Γ)
                idx = torch.full((Γ.n_G,), -1, dtype=torch.int64, device=rows.device)
                idx[rows] = torch.arange(rows.numel(), device=rows.device)
                pairs.append((ψ[ik].to(torch.complex128).contiguous(), dst, idx, None, n * nb))
            out.append(dst)
        sphere_remap(bs.architecture.ctx, pairs)
        return out
    (arg,) = args
    if isinstance(arg, PlaneWaveBasis):
        _single_rank(arg, "cell_to_supercell")
        return _supercell_basis(arg)
    scfres = arg
    _single_rank(scfres["basis"], "cell_to_supercell")
    _no_hubbard(scfres["basis"].model)
    from .densities import compute_density
    from .hamiltonian import energy_hamiltonian
    from .occupation import compute_occupation
    su = unfold_bz(scfres)
    basis = su["basis"]
    bs = _supercell_basis(basis)
    ψs = cell_to_supercell(su["psi"], basis, bs)
    eigs, psi = [], []
    for Γ, ψΓ in zip(bs.kpoints, ψs):
        e = np.concatenate([su["eigenvalues"][ik] for ik, kp in enumerate(basis.kpoints) if kp.spin == Γ.spin])
        perm = np.argsort(e, kind="stable")
        eigs.append(e[perm])
        psi.append(ψΓ[torch.as_tensor(perm, device=ψΓ.device)].contiguous())
    occ, eF = compute_occupation(bs, eigs, eF=scfres["eF"])
    rho = compute_density(bs, psi, occ, occupation_threshold=scfres.get("occupation_threshold", 0.0))
    energies, ham = energy_hamiltonian(bs, psi, occ, rho=rho, eigenvalues=eigs, eF=eF)
    return dict(scfres, ham=ham, basis=bs, psi=psi, energies=energies, rho=rho, eigenvalues=eigs, occupation=occ,
                eigenvalues_global=eigs, occupation_global=occ)
