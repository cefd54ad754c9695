"""GPU tests of the basis transfers (transfer.py over dftk_b200_remap_tables / sphere_remap / fourier_block_copy /
bspline2_*): transfers between cutoffs and the warm start they give, unfold_bz on a non-symmorphic crystal and on a spin-
polarised metal, cell_to_supercell of whole SCF results, and interpolate_density against the NumPy restatement and scipy."""
import math

import numpy as np
import pytest
import torch
from scipy import ndimage

import transfer_oracle as T
from silicon import LATTICE, POSITIONS

pytestmark = pytest.mark.gpu


def _si(dftk, symmetries=True):
    Si = dftk.ElementPsp("Si")
    return dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), symmetries=symmetries)


def _fe(dftk):
    Fe = dftk.ElementPsp("Fe", functional="pbe")
    lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
    return dftk.model_DFT(lat, [Fe], [[0, 0, 0]], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0])


def _odd(fs):
    return tuple(n + 1 - n % 2 for n in fs)


# ------------------------------------------------------------------ transfer between cutoffs
@pytest.mark.parametrize("explicit", [False, True])
def test_transfer_between_cutoffs(explicit):
    import dftk_b200 as dftk
    model = _si(dftk)
    kw = lambda E: dict(fft_size=_odd(dftk.compute_fft_size(model, E))) if explicit else {}
    b8 = dftk.PlaneWaveBasis(model, Ecut=8, kgrid=(3, 3, 3), **kw(8))
    b12 = dftk.PlaneWaveBasis(model, Ecut=12, kgrid=(3, 3, 3), **kw(12))
    psi = [dftk.random_orbitals(b8, kp, 6).contiguous() for kp in b8.kpoints]
    up = dftk.transfer_blochwave(psi, b8, b12)
    back = dftk.transfer_blochwave(up, b12, b8)
    for p, q in zip(psi, back):
        assert torch.equal(p, q)
    for p, u, k8, k12 in zip(psi, up, b8.kpoints, b12.kpoints):       # the kernels against the restatement, exactly
        ref = T.transfer_blochwave_kpt(p.cpu().numpy().T, k8.G_vectors.cpu().numpy(), k8.coordinate, b12.fft_size,
                                       k12.mapping.cpu().numpy(), k12.coordinate)
        assert np.array_equal(u.cpu().numpy().T, ref)
        i, o = dftk.transfer_mapping(b8, k8, b12, k12)
        ri, ro = T.transfer_mapping_kpt(k8.G_vectors.cpu().numpy(), k8.coordinate, b12.fft_size, k12.mapping.cpu().numpy(),
                                        k12.coordinate)
        assert np.array_equal(i.cpu().numpy(), ri) and np.array_equal(o.cpu().numpy(), ro)
    occ = [np.array([2.0, 2.0, 1.5, 0.5, 0.0, 0.0])] * len(psi)
    rho8 = dftk.compute_density(b8, psi, occ)
    rho_t = dftk.transfer_density(rho8, b8, b12)
    f8 = b8.fft(rho8).cpu().numpy()
    ref = np.real(np.fft.ifftn(T.block_copy(f8, b8.fft_size, b12.fft_size).reshape(-1, *b12.fft_size[::-1]),
                               axes=(1, 2, 3)).reshape(f8.shape[0], -1)) * b12.N * b12.ifft_normalization
    np.testing.assert_allclose(rho_t.cpu().numpy(), ref, rtol=0, atol=1e-14 * np.abs(ref).max() * 10)
    if all(n % 2 for n in b8.fft_size):
        rho12 = dftk.compute_density(b12, up, occ)
        assert (rho12 - rho_t).abs().max().item() < 1e-12


def test_warm_start_from_a_lower_cutoff():
    import dftk_b200 as dftk
    model = _si(dftk)
    b8 = dftk.PlaneWaveBasis(model, Ecut=8, kgrid=(3, 3, 3))
    b12 = dftk.PlaneWaveBasis(model, Ecut=12, kgrid=(3, 3, 3))
    r8 = dftk.self_consistent_field(b8, tol=1e-10)
    cold = dftk.self_consistent_field(b12, tol=1e-10)
    warm = dftk.self_consistent_field(b12, tol=1e-10, psi=dftk.transfer_blochwave(r8["psi"], b8, b12),
                                      rho=dftk.transfer_density(r8["rho"], b8, b12))
    print(f"SCF iterations at Ecut 12: cold start {cold['n_iter']}, warm start from Ecut 8 {warm['n_iter']}")
    assert cold["converged"] and warm["converged"]
    assert abs(warm["energies"].total - cold["energies"].total) < 1e-8
    assert warm["n_iter"] <= cold["n_iter"]


# ------------------------------------------------------------------ unfold_bz
def _residuals(ham, psi, eigs):
    out = []
    for ik, (p, e) in enumerate(zip(psi, eigs)):
        hp = ham[ik].mul(p)
        r = hp - torch.as_tensor(e, device=p.device)[:, None] * p
        out.append(r.norm(dim=1).cpu().numpy())
    return out


def _check_unfold(dftk, scfres, nconv):
    from dftk_b200.device import density_accumulate_multi
    su = dftk.unfold_bz(scfres)
    bu, b = su["basis"], scfres["basis"]
    assert len(bu.kpoints) == len(b.kgrid) * b.model.n_spin_components and bu.fft_size == b.fft_size
    assert len(bu.symmetries) == len(b.symmetries)
    assert abs(su["energies"].total - scfres["energies"].total) < 1e-10
    _, ham_u = dftk.energy_hamiltonian(bu, su["psi"], su["occupation"], rho=scfres["rho"], eigenvalues=su["eigenvalues"],
                                       eF=scfres["eF"])
    e_u = dftk.energy(bu, su["psi"], su["occupation"], rho=scfres["rho"], eigenvalues=su["eigenvalues"], eF=scfres["eF"])
    assert abs(e_u.total - scfres["energies"].total) < 1e-10
    rho = torch.zeros_like(scfres["rho"])        # accumulated WITHOUT symmetrisation: tests the phase convention of τ
    density_accumulate_multi(bu.kblocks, [p.contiguous() for p in su["psi"]],
                             [np.asarray(o) * w for o, w in zip(su["occupation"], bu.kweights)], rho)
    assert (rho - scfres["rho"]).abs().max().item() < 1e-10
    r0 = max(r[:nconv].max() for r in _residuals(scfres["ham"], scfres["psi"], scfres["eigenvalues"]))
    r1 = max(r[:nconv].max() for r in _residuals(su["ham"], su["psi"], su["eigenvalues"]))
    assert r1 <= 10 * r0 + 1e-12, (r0, r1)
    return su


def test_unfold_bz_silicon_nonsymmorphic():
    import dftk_b200 as dftk
    model = _si(dftk)
    assert any(np.any(np.abs(s.tau) > 1e-12) for s in model.symmetries)
    b = dftk.PlaneWaveBasis(model, Ecut=8, kgrid=(4, 4, 4))
    assert len(b.kpoints) < 64
    r = dftk.self_consistent_field(b, tol=1e-10)
    su = _check_unfold(dftk, r, 4)
    bn = dftk.PlaneWaveBasis(_si(dftk, symmetries=False), Ecut=8, kgrid=(4, 4, 4), fft_size=b.fft_size)
    rn = dftk.self_consistent_field(bn, tol=1e-10)
    for ku, eu in zip(su["basis"].kpoints, su["eigenvalues"]):
        j = [i for i, kp in enumerate(bn.kpoints) if np.allclose(kp.coordinate, ku.coordinate)][0]
        np.testing.assert_allclose(eu[:4], rn["eigenvalues"][j][:4], rtol=0, atol=1e-6)


def test_unfold_bz_iron_collinear():
    import dftk_b200 as dftk
    b = dftk.PlaneWaveBasis(_fe(dftk), Ecut=15, kgrid=(3, 3, 3))
    r = dftk.self_consistent_field(b, tol=1e-9, mixing=dftk.KerkerMixing())
    _check_unfold(dftk, r, 4)


# ------------------------------------------------------------------ cell_to_supercell
def _check_supercell(dftk, r, rep, n_cells):
    rs = dftk.cell_to_supercell(r)
    bs = rs["basis"]
    assert len(bs.kpoints) == r["basis"].model.n_spin_components and bs.fft_size == tuple(n * rep for n in r["basis"].fft_size)
    for p in rs["psi"]:
        G = p @ p.conj().T
        assert (G - torch.eye(G.shape[0], dtype=G.dtype, device=G.device)).abs().max().item() < 1e-13
    nx, ny, nz = r["basis"].fft_size
    tiled = r["rho"].reshape(-1, nz, ny, nx).repeat(1, rep, rep, rep).reshape(r["rho"].shape[0], -1)
    assert (rs["rho"] - tiled).abs().max().item() < 1e-10
    itp = dftk.interpolate_density(r["rho"], r["basis"], bs)
    assert torch.equal(itp, tiled)
    assert abs(rs["energies"].total - n_cells * r["energies"].total) < 1e-9 * n_cells
    step = dftk.self_consistent_field(bs, psi=rs["psi"], rho=rs["rho"], maxiter=1, tol=1e-12)
    assert abs(step["energies"].total - rs["energies"].total) < 1e-8 * n_cells
    return rs


# The unit SCF symmetrises its density on its own grid, which commutes with unfolding only when the grid holds the density's
# spectrum: Ecut 8 needs 24 points per axis (at 18 the aliased products leave ρ_unit 1e-7 away from the unfolded sum).
@pytest.mark.parametrize("rep,Ecut,fft", [(2, 8, 24), (3, 12, 24)])
def test_cell_to_supercell_silicon(rep, Ecut, fft):
    import dftk_b200 as dftk
    bu = dftk.PlaneWaveBasis(_si(dftk), Ecut=Ecut, kgrid=(rep,) * 3, fft_size=(fft,) * 3)
    assert len(bu.kpoints) < rep ** 3
    ru = dftk.self_consistent_field(bu, tol=1e-10)
    _check_supercell(dftk, ru, rep, rep ** 3)


def test_cell_to_supercell_iron_collinear():
    import dftk_b200 as dftk
    b = dftk.PlaneWaveBasis(_fe(dftk), Ecut=15, kgrid=(2, 2, 2))
    r = dftk.self_consistent_field(b, tol=1e-10, mixing=dftk.KerkerMixing())
    _check_supercell(dftk, r, 2, 8)


def test_cell_to_supercell_refuses_a_shifted_grid():
    import dftk_b200 as dftk
    b = dftk.PlaneWaveBasis(_si(dftk), Ecut=5, kgrid=(2, 2, 2), kshift=(0.5, 0.5, 0.5))
    with pytest.raises(NotImplementedError):
        dftk.cell_to_supercell(b)


# ------------------------------------------------------------------ interpolate_density
def _smooth(grid, seed):
    nx, ny, nz = grid
    Z, Y, X = np.meshgrid(np.arange(nz) / nz, np.arange(ny) / ny, np.arange(nx) / nx, indexing="ij")
    f = 1.0 + 0.1 * np.random.default_rng(seed).random((nz, ny, nx))
    return f + np.cos(2 * math.pi * (X + 2 * Y)) + 0.5 * np.sin(2 * math.pi * (Z - X))


@pytest.mark.parametrize("grid_in,grid_out", [((12, 12, 12), (18, 18, 18)), ((18, 18, 18), (12, 12, 12)),
                                              ((18, 20, 24), (25, 27, 30)), ((25, 27, 30), (18, 20, 24)),
                                              ((150, 150, 150), (96, 96, 96)), ((150, 150, 150), (192, 192, 192))])
def test_interpolate_density_device(grid_in, grid_out):
    import dftk_b200 as dftk
    f = np.stack([_smooth(grid_in, 1), _smooth(grid_in, 2)])
    out = dftk.interpolate_density(torch.as_tensor(f, device="cuda"), grid_out).cpu().numpy()
    nxo, nyo, nzo = grid_out
    Z, Y, X = np.meshgrid(np.arange(nzo), np.arange(nyo), np.arange(nxo), indexing="ij")
    coords = [Z * grid_in[2] / nzo, Y * grid_in[1] / nyo, X * grid_in[0] / nxo]
    for s in range(2):
        ref = ndimage.map_coordinates(f[s], coords, order=2, mode="grid-wrap")
        np.testing.assert_allclose(out[s], ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
        if grid_in[0] < 100:
            ref = T.interpolate_density(f[s], grid_out)
            np.testing.assert_allclose(out[s], ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
    same = dftk.interpolate_density(torch.as_tensor(f, device="cuda"), grid_in).cpu().numpy()
    assert np.array_equal(same, f)


def test_interpolate_density_supercell_form():
    import dftk_b200 as dftk
    f = _smooth((9, 10, 8), 3)[None]
    lat = np.diag([4.0, 5.0, 3.5])
    out = dftk.interpolate_density(torch.as_tensor(f, device="cuda"), (9, 10, 8), (20, 17, 24), lat, lat @ np.diag([2, 2, 3]))
    ref = T.interpolate_density(f[0], (20, 17, 24), rep=(2, 2, 3))
    np.testing.assert_allclose(out.cpu().numpy()[0], ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
