"""The fused y-z stage of the local H apply (kr_yz_apply, fft_reg.cuh) on the device against the direct DFT of
tests/fft_reference.py.

kb_apply_local_kinetic (fft.cu) takes the fused path when all three axes have a factor pair of the register engine, the
sphere has the range form, ny == nz and the y-z intermediate of one x line fits in a CTA's shared memory.  Every pair runs
on an (18, n, n) box with a half and a full off-centre ellipsoid; `_fused` mirrors the rule and the launch count shows
which path ran (three kernels per band chunk fused, five otherwise).  A 150^3 block with the Γ sphere of the benchmark's
128-atom silicon cell is checked as well.
"""
import numpy as np
import pytest
import torch

import fft_reference as fr

pytestmark = pytest.mark.gpu

PAIR_OF = {a * b: (a, b) for a, b in fr.reg_pairs()}
NX = 18
TOL = 1e-13
NB = 5
YZ_LINES = 25                                # RegYZ<A,B>::LL


def _fused(shape, mapping, smem_optin):
    """Mirror of kb_yz_fused (fft.cu)."""
    nx, ny, nz = shape
    if not (nx in PAIR_OF and ny in PAIR_OF and nz in PAIR_OF and ny == nz):
        return False
    n_zc = np.unique(mapping // (nx * ny)).size
    return (n_zc + YZ_LINES) * (ny | 1) * 16 <= smem_optin


def _crand(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _check(got, ref):
    err = float(np.abs(got.cpu().numpy() - ref).max() / np.abs(ref).max())
    assert err <= TOL, err


def _local_launches(c, kb, d):
    c.launch_count(reset=True)
    kb.apply_terms(d, 1)
    return c.launch_count()


def _apply_checks(c, kb, psi, V, mapping, shape, kin, rng):
    from gpu_common import to_dev
    loc = fr.local_apply(psi, mapping, shape, V)
    full = loc + kin * psi
    d = to_dev(psi[:3])
    _check(kb.apply_terms(d, 1), loc[:3])
    _check(kb.apply_terms(d, 3), full[:3])
    out0 = _crand(rng, 3, mapping.size)
    out = to_dev(out0)
    kb.apply_terms(d, 3, out=out, accumulate=True)
    _check(out, out0 + full[:3])
    _check(kb.apply_terms(to_dev(psi[:1]), 3), full[:1])
    c.set_option("band_chunk", 2)
    try:
        _check(kb.apply_terms(to_dev(psi), 3), full)
    finally:
        c.set_option("band_chunk", 0)


@pytest.mark.parametrize("n", sorted(PAIR_OF))
def test_yz_fused_every_pair(n):
    import dftk_b200
    from gpu_common import ctx, to_dev
    c = ctx()
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    shape = (NX, n, n)
    N = NX * n * n
    rng = np.random.default_rng(n)
    V = rng.standard_normal(N)
    grid = dftk_b200.FFTGrid(c, shape, 7.3)
    took = {}
    for frac in (fr.HALF, fr.FULL):
        mp = fr.ellipsoid_mapping(shape, frac)
        kin = rng.random(mp.size)
        psi = _crand(rng, NB, mp.size)
        kb = dftk_b200.KBlock(grid, mp, kin=kin)
        kb.set_potential(to_dev(V))
        fused = _fused(shape, mp, optin)
        assert _local_launches(c, kb, to_dev(psi[:3])) == (3 if fused else 5)
        took[frac] = fused
        _apply_checks(c, kb, psi, V, mp, shape, kin, rng)
        # the SCF's shared grid potential (its [x][y][z] copy is written by grid_set_potential)
        Vg = rng.standard_normal(N)
        grid.set_potential(0, to_dev(Vg))
        kb.use_grid_potential(0)
        _check(kb.apply_terms(to_dev(psi[:3]), 3), fr.local_apply(psi[:3], mp, shape, Vg, kin))
    # in the 227 KiB of an H100 CTA: the half sphere's intermediate up to n = 144, the whole box up to n = 108
    assert took[fr.HALF] == (n <= 144)
    assert took[fr.FULL] == (n <= 108)


def test_yz_unfused_shapes_keep_five_stages():
    """ny != nz, and an axis without a factor pair: the five-kernel path."""
    import dftk_b200
    from gpu_common import ctx, to_dev
    c = ctx()
    rng = np.random.default_rng(1)
    for shape in [(18, 25, 30), (18, 14, 14)]:
        N = int(np.prod(shape))
        V = rng.standard_normal(N)
        mp = fr.ellipsoid_mapping(shape, fr.HALF)
        psi = _crand(rng, 3, mp.size)
        kb = dftk_b200.KBlock(dftk_b200.FFTGrid(c, shape, 7.3), mp, kin=rng.random(mp.size))
        kb.set_potential(to_dev(V))
        assert not _fused(shape, mp, torch.cuda.get_device_properties(0).shared_memory_per_block_optin)
        assert _local_launches(c, kb, to_dev(psi)) == 5
        _check(kb.apply_terms(to_dev(psi), 1), fr.local_apply(psi, mp, shape, V))


def test_yz_fused_bench_cell_gamma_sphere():
    """150^3 grid with the Γ sphere of the 128-atom Si cell at Ecut = 30 Ha (n_pw = 135 491, 71 z planes)."""
    import dftk_b200
    from gpu_common import ctx, to_dev
    c = ctx()
    n = 150
    a = 10.26 / 2
    lattice = 4 * np.array([[0, a, a], [a, 0, a], [a, a, 0]])
    recip = 2 * np.pi * np.linalg.inv(lattice).T
    g = fr.centred_freqs(n)
    gz, gy, gx = np.meshgrid(g, g, g, indexing="ij")
    G = np.stack([gx, gy, gz], -1) @ recip.T
    mp = np.flatnonzero(((G ** 2).sum(-1) / 2 <= 30.0).reshape(-1)).astype(np.int64)
    assert mp.size == 135491 and np.unique(mp // (n * n)).size == 71
    shape = (n, n, n)
    assert _fused(shape, mp, torch.cuda.get_device_properties(0).shared_memory_per_block_optin)
    rng = np.random.default_rng(150)
    V = rng.standard_normal(n ** 3)
    kin = rng.random(mp.size)
    psi = _crand(rng, 2, mp.size)
    kb = dftk_b200.KBlock(dftk_b200.FFTGrid(c, shape, 7.3), mp, kin=kin)
    kb.set_potential(to_dev(V))
    assert _local_launches(c, kb, to_dev(psi)) == 3
    _check(kb.apply_terms(to_dev(psi), 3), fr.local_apply(psi, mp, shape, V, kin))
