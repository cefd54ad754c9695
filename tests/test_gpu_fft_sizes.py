"""Every FFT axis length of the k-point pipeline on the device against the direct DFT of tests/fft_reference.py.

Each factor pair of the register two-pass engine (DFTK_REG_PAIRS, fft_plan.h) and a set of lengths of the generic
Stockham engine is placed on x, y and z of an (n, 18, 25)-type box.  Under both FFT engines (option fft_engine) every
stage is compared with the reference: local and kinetic apply (also accumulating, with z_pipeline 0 and 1, one band and
chunked bands), sphere -> real, real -> sphere, density, and the cube FFT.  The batched kernels of lobpcg_multi and
density_accumulate_multi are checked on three k-blocks of different sizes, spins and potentials on one grid.

Run with -s to see the largest error per stage and engine and which (axis, engine, z_pipeline) combinations ran; set
DFTK_FFT_SWEEP_REPORT to a file name to also get them as JSON.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

import fft_reference as fr

pytestmark = pytest.mark.gpu

PAIR_OF = {a * b: (a, b) for a, b in fr.reg_pairs()}
REG_LENGTHS = sorted(PAIR_OF)
# lengths without a factor pair: 5-smooth ones, ones above 256, ones with a factor 7, 11 or 13, and a large prime
GENERIC_LENGTHS = [50, 81, 162, 243, 250, 270, 288, 320, 384, 400, 512, 14, 22, 26, 49, 77, 91, 97]
assert not set(GENERIC_LENGTHS) & set(REG_LENGTHS)
SHAPES = [(n, ax) for n in REG_LENGTHS + GENERIC_LENGTHS for ax in "xyz"]
# the batched kernels: every pair on z, a subset on x and y
BATCH_XY = sorted(set(REG_LENGTHS[::4]) | {150, 192})
BATCH_SHAPES = [(n, "z") for n in REG_LENGTHS] + [(n, ax) for n in BATCH_XY for ax in "xy"]
VOLUME = 7.3
TOL = 1e-13
NB = 5                                      # bands of the references; the plain calls use the first three
WEIGHTS = np.array([1.0, 0.0, 2.5, 0.5, 0.0])

_ERR = {}                                   # (stage, engine) -> largest |got - ref| / max|ref|
_RAN = set()                                # (n, axis, engine, z_pipeline) of the stage sweep
_PIPE = set()                               # (n, axis) where the persistent z stage was taken


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if not _ERR:
        return
    print("\nlargest |device - direct DFT| / max|reference|:")
    for (stage, engine), v in sorted(_ERR.items()):
        print(f"  {stage:34s} engine {engine}: {v:.2e}")
    full = [n for n in REG_LENGTHS
            if all((n, ax, e, zp) in _RAN for ax in "xyz" for e in (0, 1) for zp in (0, 1))]
    print(f"register pairs run on x, y and z under both engines with z_pipeline 0 and 1: {len(full)} of {len(REG_LENGTHS)}")
    print(f"shapes where the persistent z stage ran: {len(_PIPE)}")
    path = os.environ.get("DFTK_FFT_SWEEP_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(max_rel_err={f"{s} engine {e}": v for (s, e), v in sorted(_ERR.items())},
                           pairs_complete=len(full), pairs=len(REG_LENGTHS), ran=sorted(map(list, _RAN)),
                           pipe_shapes=sorted(map(list, _PIPE))), f, indent=1)


def _check(stage, engine, got, ref):
    if isinstance(got, torch.Tensor):
        got = got.cpu().numpy()
    err = float(np.abs(got - ref).max() / np.abs(ref).max())
    _ERR[(stage, engine)] = max(_ERR.get((stage, engine), 0.0), err)
    assert err <= TOL, (stage, engine, err)


def _kin(shape, mapping, k):
    """|G + k|^2 / 2 of a box cell with grid spacing 0.25 bohr."""
    nx, ny, nz = shape
    iz, iy, ix = np.unravel_index(mapping, (nz, ny, nx))
    return 0.5 * sum((2 * np.pi * (fr.centred_freqs(n)[i] + ki) / (0.25 * n)) ** 2
                     for n, i, ki in ((nx, ix, k[0]), (ny, iy, k[1]), (nz, iz, k[2])))


def _crand(rng, *shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


def _pipe_bands(shape, mapping, sm_count):
    """Band count for which kb_apply_local_kinetic (fft.cu) runs the persistent cp.async z stage (z_apply_pipe) with
    z_pipeline = 1, or None when the z axis has no factor pair.  Mirrors the condition there: shared memory of the
    pipelined stage <= 100 KiB and at least two tiles per SM."""
    nx, ny, nz = shape
    if nz not in PAIR_OF:
        return None
    a, b = PAIR_OF[nz]
    t = max(a, b)
    L = 8 if t >= 12 else (16 if t >= 5 else 32)
    n_zc = np.unique(mapping // (nx * ny)).size
    sm_pipe = a * b * (L + 1) * 16 + 2 * n_zc * L * 16
    tiles_per_band = -(-nx // L) * ny
    nb = -(-2 * sm_count // tiles_per_band)
    assert sm_pipe <= 100 * 1024 and tiles_per_band * nb >= 2 * sm_count
    return nb


def _sphere_case(shape, frac, V, rng):
    mp = fr.ellipsoid_mapping(shape, frac)
    N = int(np.prod(shape))
    assert frac != fr.FULL or mp.size == N
    kin = _kin(shape, mp, fr.K_OFF)
    psi = _crand(rng, NB, mp.size)
    f = _crand(rng, NB, N)
    cube = fr.sphere_to_real(psi, mp, shape)
    return dict(name="half" if frac == fr.HALF else "full", mapping=mp, kin=kin, psi=psi, f=f, out0=_crand(rng, 3, mp.size),
                loc=fr.local_apply(psi, mp, shape, V), cube=cube, back=fr.real_to_sphere(f, mp, shape),
                rho0=rng.random(N), rho=(WEIGHTS[:, None] * np.abs(cube) ** 2).sum(0) / VOLUME)


def _apply_checks(kb, case, engine, tag):
    from gpu_common import to_dev
    psi, kin, loc = case["psi"], case["kin"], case["loc"]
    full = loc + kin * psi
    d = to_dev(psi[:3])
    _check(f"apply local{tag}", engine, kb.apply_terms(d, 1), loc[:3])
    _check(f"apply local+kin{tag}", engine, kb.apply_terms(d, 3), full[:3])
    out = to_dev(case["out0"])
    kb.apply_terms(d, 3, out=out, accumulate=True)
    _check(f"apply accumulate{tag}", engine, out, case["out0"] + full[:3])
    _check(f"apply 1 band{tag}", engine, kb.apply_terms(to_dev(psi[:1]), 3), full[:1])
    kb.ctx.set_option("band_chunk", 2)
    try:
        _check(f"apply chunk 2 of 5{tag}", engine, kb.apply_terms(to_dev(psi), 3), full)
    finally:
        kb.ctx.set_option("band_chunk", 0)


def _transform_checks(kb, case, engine):
    from gpu_common import to_dev
    ifn, ffn = 1 / math.sqrt(VOLUME), math.sqrt(VOLUME) / kb.grid.N
    psi, cube, back = case["psi"], case["cube"], case["back"]
    d = to_dev(psi[:3])
    _check("sphere_to_real", engine, kb.sphere_to_real(d, normalize=True), ifn * cube[:3])
    _check("sphere_to_real unnormalised", engine, kb.sphere_to_real(d, normalize=False), cube[:3])
    _check("sphere_to_real 1 band", engine, kb.sphere_to_real(to_dev(psi[:1])), ifn * cube[:1])
    f = to_dev(case["f"][:3])
    _check("real_to_sphere", engine, kb.real_to_sphere(f, normalize=True), ffn * back[:3])
    _check("real_to_sphere unnormalised", engine, kb.real_to_sphere(f, normalize=False), back[:3])
    rho = to_dev(case["rho0"])
    kb.density_accumulate(to_dev(psi), WEIGHTS, rho)
    _check("density", engine, rho.cpu().numpy() - case["rho0"], case["rho"])
    kb.ctx.set_option("band_chunk", 2)
    try:
        _check("sphere_to_real chunk 2 of 5", engine, kb.sphere_to_real(to_dev(psi)), ifn * cube)
        _check("real_to_sphere chunk 2 of 5", engine, kb.real_to_sphere(to_dev(case["f"])), ffn * back)
        rho = to_dev(case["rho0"])
        kb.density_accumulate(to_dev(psi), WEIGHTS, rho)
        _check("density chunk 2 of 5", engine, rho.cpu().numpy() - case["rho0"], case["rho"])
    finally:
        kb.ctx.set_option("band_chunk", 0)


@pytest.mark.parametrize("n,axis", SHAPES, ids=[f"{n}-{ax}" for n, ax in SHAPES])
def test_pipeline_stages_against_direct_dft(n, axis):
    import dftk_b200
    from gpu_common import ctx, to_dev
    c = ctx()
    shape = fr.placements(n)[axis]
    N = int(np.prod(shape))
    rng = np.random.default_rng(3 * n + "xyz".index(axis))
    V = rng.standard_normal(N)
    cases = [_sphere_case(shape, frac, V, rng) for frac in (fr.HALF, fr.FULL)]
    half = cases[0]
    nb_pipe = _pipe_bands(shape, half["mapping"], torch.cuda.get_device_properties(0).multi_processor_count)
    if nb_pipe is not None:
        psi_pipe = _crand(rng, nb_pipe, half["mapping"].size)
        ref_pipe = fr.local_apply(psi_pipe, half["mapping"], shape, V, half["kin"])
    x = _crand(rng, 2, N)
    for engine in (0, 1):
        c.set_option("fft_engine", engine)            # applies to grids created afterwards
        try:
            grid = dftk_b200.FFTGrid(c, shape, VOLUME)
        finally:
            c.set_option("fft_engine", 0)
        if engine == 0:                               # the cube FFT is the generic engine under either option
            _check("fft_cube forward", engine, grid.fft_cube(to_dev(x), -1), fr.dft3(x, shape, -1))
            _check("fft_cube backward", engine, grid.fft_cube(to_dev(x), +1), fr.dft3(x, shape, +1))
        for case in cases:
            kb = dftk_b200.KBlock(grid, case["mapping"], kin=case["kin"])
            kb.set_potential(to_dev(V))
            for zp in (0, 1):
                c.set_option("z_pipeline", zp)
                try:
                    _apply_checks(kb, case, engine, f" ({case['name']} sphere)")
                    if zp == 1 and case is half and nb_pipe is not None:
                        # engine 0: z_apply_pipe; engine 1 has no such stage and runs its own z stage
                        _check("apply at the z_apply_pipe band count", engine, kb.apply_terms(to_dev(psi_pipe), 3), ref_pipe)
                        if engine == 0:
                            _PIPE.add((n, axis))
                finally:
                    c.set_option("z_pipeline", 0)
                _RAN.add((n, axis, engine, zp))
            _transform_checks(kb, case, engine)


@pytest.mark.parametrize("shape", [(15, 18, 25), (18, 25, 150), (97, 18, 25)])
def test_one_point_sphere(shape):
    """A sphere of the single point G = 0: one column, one z plane."""
    import dftk_b200
    from gpu_common import ctx, to_dev
    c = ctx()
    N = int(np.prod(shape))
    rng = np.random.default_rng(5)
    V = rng.standard_normal(N)
    mp = fr.ellipsoid_mapping(shape, 0)
    kin = np.array([0.3])
    psi = _crand(rng, 2, 1)
    f = _crand(rng, 2, N)
    for engine in (0, 1):
        c.set_option("fft_engine", engine)
        try:
            grid = dftk_b200.FFTGrid(c, shape, VOLUME)
        finally:
            c.set_option("fft_engine", 0)
        kb = dftk_b200.KBlock(grid, mp, kin=kin)
        kb.set_potential(to_dev(V))
        _check("one-point apply", engine, kb.apply_terms(to_dev(psi), 3), fr.local_apply(psi, mp, shape, V, kin))
        _check("one-point sphere_to_real", engine, kb.sphere_to_real(to_dev(psi), normalize=False),
               fr.sphere_to_real(psi, mp, shape))
        _check("one-point real_to_sphere", engine, kb.real_to_sphere(to_dev(f), normalize=False),
               fr.real_to_sphere(f, mp, shape))
        rho = torch.zeros(N, dtype=torch.float64, device=c.device)
        kb.density_accumulate(to_dev(psi), [2.0, 0.0], rho)
        _check("one-point density", engine, rho, 2.0 * np.abs(psi[0, 0]) ** 2 / VOLUME * np.ones(N))


# three k-blocks on one grid: offsets and sphere sizes differ (so n_pw, n_cols and n_zc differ), spins 0 and 1
K_BLOCKS = [(fr.K_OFF, 0.5, 0), ((-0.35, 0.1, 0.2), 0.42, 1), ((0.0, 0.4, -0.15), 0.57, 0)]


@pytest.mark.parametrize("n,axis", BATCH_SHAPES, ids=[f"{n}-{ax}" for n, ax in BATCH_SHAPES])
def test_batched_kernels(n, axis):
    """density_accumulate_multi against the reference for a (2, N) density; lobpcg_multi against per-block lobpcg
    (same arguments, two iterations), and its eigenvalues against Rayleigh quotients taken with apply_terms.  Every block
    has its own potential, so items that borrow another item's data are noticed."""
    import dftk_b200
    from dftk_b200.device import density_accumulate_multi, lobpcg_multi
    from gpu_common import ctx, to_dev
    c = ctx()
    shape = fr.placements(n)[axis]
    nx, ny, nz = shape
    N = int(np.prod(shape))
    rng = np.random.default_rng(7 * n + "xyz".index(axis))
    grid = dftk_b200.FFTGrid(c, shape, VOLUME)
    kbs, maps = [], []
    for k, frac, spin in K_BLOCKS:
        mp = fr.ellipsoid_mapping(shape, frac, k)
        kb = dftk_b200.KBlock(grid, mp, kin=_kin(shape, mp, k), spin=spin)
        kb.set_potential(to_dev(rng.standard_normal(N)))
        kbs.append(kb)
        maps.append(mp)
    assert len({m.size for m in maps}) == 3
    assert len({np.unique(m // nx).size for m in maps}) == 3            # n_cols
    assert len({np.unique(m // (nx * ny)).size for m in maps}) == 3     # n_zc
    # density of blocks with 4, 2 and 3 bands into the channel of their spin
    weights = [np.array([2.0, 0.0, 1.0, 0.5]), np.array([0.0, 1.5]), np.array([0.25, 1.0, 0.0])]
    psis = [_crand(rng, len(w), m.size) for w, m in zip(weights, maps)]
    rho0 = rng.random((2, N))
    ref = np.zeros((2, N))
    for (_, _, spin), w, p, m in zip(K_BLOCKS, weights, psis, maps):
        ref[spin] += fr.density(p, w, m, shape, 1 / math.sqrt(VOLUME))
    rho = to_dev(rho0)
    density_accumulate_multi(kbs, [to_dev(p) for p in psis], weights, rho)
    _check("density_accumulate_multi", 0, rho.cpu().numpy() - rho0, ref)
    # two LOBPCG iterations of all blocks at once == the same iterations block by block
    nb = 4
    X0 = [_crand(rng, nb, m.size) for m in maps]
    single = [kb.lobpcg(to_dev(x), tol=1e-14, miniter=2, maxiter=2) for kb, x in zip(kbs, X0)]
    multi = lobpcg_multi(kbs, [to_dev(x) for x in X0], tol=1e-14, miniter=2, maxiter=2)
    for kb, rs, rm in zip(kbs, single, multi):
        assert rs["n_iter"] == rm["n_iter"] and rs["n_matvec"] == rm["n_matvec"]
        scale = max(1.0, np.abs(rs["λ"]).max())
        np.testing.assert_allclose(rm["λ"], rs["λ"], rtol=0, atol=1e-10 * scale)
        Xs, Xm = rs["X"].cpu().numpy(), rm["X"].cpu().numpy()
        phase = np.sum(Xs.conj() * Xm, axis=1)
        phase /= np.abs(phase)
        np.testing.assert_allclose(Xm, phase[:, None] * Xs, rtol=0, atol=1e-10)
        HX = kb.apply_terms(rm["X"], 3).cpu().numpy()
        rq = np.real(np.sum(Xm.conj() * HX, axis=1)) / np.sum(np.abs(Xm) ** 2, axis=1)
        np.testing.assert_allclose(rm["λ"], rq, rtol=0, atol=1e-10 * scale)
