"""GPU parity tests of every kernel family against the CPU oracle (run on an H100: -m gpu).
All calls go through the C ABI (ctypes)."""
import os
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def si():
    from gpu_common import silicon_setup, device_blocks
    m, b, t, rho, ham = silicon_setup()
    grid, blocks = device_blocks(b, ham)
    return dict(m=m, b=b, t=t, rho=rho, ham=ham, grid=grid, kb=blocks[0], blk=ham[0])


@pytest.mark.parametrize("fft_size", [(8, 9, 10), (27, 27, 27), (40, 40, 40), (33, 20, 17), (48, 45, 32)])
def test_fft_cube(fft_size):
    import dftk_b200
    from gpu_common import ctx, to_dev
    nx, ny, nz = fft_size
    grid = dftk_b200.FFTGrid(ctx(), fft_size, 10.0)
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, nz, ny, nx)) + 1j * rng.standard_normal((2, nz, ny, nx))
    for sign in (-1, 1):
        d = to_dev(x.reshape(2, -1))
        grid.fft_cube(d, sign)
        ref = np.fft.fftn(x, axes=(1, 2, 3)) if sign < 0 else np.fft.ifftn(x, axes=(1, 2, 3)) * (nx * ny * nz)
        np.testing.assert_allclose(d.cpu().numpy().reshape(x.shape), ref, atol=1e-12 * np.abs(ref).max())


def test_sphere_transforms(si):
    from gpu_common import to_dev, rand_psi
    b, kb, kpt = si["b"], si["kb"], si["blk"].kpt
    psi = rand_psi(kpt.n_G, 5)
    out = kb.sphere_to_real(to_dev(psi), normalize=True).cpu().numpy()
    ref = np.stack([b.ifft_kpt(kpt, p) for p in psi])
    np.testing.assert_allclose(out, ref, atol=1e-12 * np.abs(ref).max())
    rng = np.random.default_rng(3)
    f = rng.standard_normal((3, b.N)) + 1j * rng.standard_normal((3, b.N))
    back = kb.real_to_sphere(to_dev(f), normalize=True).cpu().numpy()
    refb = np.stack([b.fft_kpt(kpt, x) for x in f])
    np.testing.assert_allclose(back, refb, atol=1e-12 * np.abs(refb).max())
    # round trip (test/fourier_transforms.jl:1-47)
    rt = kb.real_to_sphere(kb.sphere_to_real(to_dev(psi))).cpu().numpy()
    np.testing.assert_allclose(rt, psi, atol=1e-12)


@pytest.mark.parametrize("backend", [0, 1])
def test_apply_h_terms(si, backend):
    from gpu_common import to_dev, rand_psi, ctx
    ctx().set_option("gemm_backend", backend)
    try:
        blk, kb = si["blk"], si["kb"]
        psi = rand_psi(blk.kpt.n_G, 7, seed=1)
        d = to_dev(psi)
        P, D = blk.PD
        ref_loc = blk.local_apply(psi.T).T
        ref_kin = blk.kin[None, :] * psi
        ref_nl = (P @ (D @ (P.conj().T @ psi.T))).T
        scale = np.abs(ref_loc + ref_kin + ref_nl).max()
        np.testing.assert_allclose(kb.apply_terms(d, 1).cpu().numpy(), ref_loc, atol=1e-12 * scale)
        np.testing.assert_allclose(kb.apply_terms(d, 2).cpu().numpy(), ref_kin, atol=1e-12 * scale)
        np.testing.assert_allclose(kb.apply_terms(d, 4).cpu().numpy(), ref_nl, atol=1e-12 * scale)
        np.testing.assert_allclose(kb.apply_h(d).cpu().numpy(), blk.matmul(psi.T).T, atol=1e-12 * scale)
        # accumulate semantics of apply! (src/terms/operators.jl:6-8)
        acc = to_dev(psi.copy())
        kb.apply_terms(d, 7, out=acc, accumulate=True)
        np.testing.assert_allclose(acc.cpu().numpy(), psi + blk.matmul(psi.T).T, atol=1e-12 * scale)
        # host buffers through the same C ABI call (end-to-end path)
        hout = np.zeros_like(psi)
        from dftk_b200._lib import check
        from dftk_b200.device import _ptr
        check(kb.ctx.L.dftk_b200_apply_h(kb.h, _ptr(psi), _ptr(hout), psi.shape[0]), kb.ctx.h)
        np.testing.assert_allclose(hout, blk.matmul(psi.T).T, atol=1e-12 * scale)
    finally:
        ctx().set_option("gemm_backend", 0)


@pytest.mark.parametrize("shape", [(1000, 7, 5), (4099, 70, 33), (129, 64, 32), (20000, 130, 1), (515, 3, 97)])
def test_zgemm_own_kernels(shape):
    from gpu_common import ctx
    K, m, n = shape
    c = ctx()
    g = torch.Generator(device="cpu").manual_seed(0)
    A = torch.randn(m, K, 2, generator=g, dtype=torch.float64)
    B = torch.randn(n, K, 2, generator=g, dtype=torch.float64)
    A = torch.view_as_complex(A).to(c.device)
    B = torch.view_as_complex(B).to(c.device)
    C0 = torch.view_as_complex(torch.randn(n, m, 2, generator=g, dtype=torch.float64)).to(c.device)
    alpha, beta = 0.7 - 0.2j, -0.3 + 1.1j
    # Gram: C(m x n) = A^H B ; tensors are stored (cols, rows)
    C = C0.clone()
    c.zgemm("C", A, B, C, alpha, beta)
    ref = alpha * (B @ A.conj().T) + beta * C0      # (n, m) = column-major m x n
    assert (C - ref).abs().max().item() < 1e-11 * ref.abs().max().item()
    # update: X(K x n) = A(K x m) * S(m x n)
    S = torch.view_as_complex(torch.randn(n, m, 2, generator=g, dtype=torch.float64)).to(c.device)
    X0 = torch.view_as_complex(torch.randn(n, K, 2, generator=g, dtype=torch.float64)).to(c.device)
    X = X0.clone()
    c.zgemm("N", A, S, X, alpha, beta)
    refx = alpha * (S @ A) + beta * X0
    assert (X - refx).abs().max().item() < 1e-11 * refx.abs().max().item()


def test_band_energies_and_density(si):
    from gpu_common import to_dev, rand_psi, ctx
    b, blk, kb = si["b"], si["blk"], si["kb"]
    psi = rand_psi(blk.kpt.n_G, 6, seed=4)
    ek, en = kb.band_energies(to_dev(psi))
    P, D = blk.PD
    Pp = P.conj().T @ psi.T
    np.testing.assert_allclose(ek, np.real(np.sum(np.conj(psi) * blk.kin[None, :] * psi, axis=1)), rtol=1e-12)
    np.testing.assert_allclose(en, np.sum(np.real(np.conj(Pp) * (D @ Pp)), axis=0), rtol=1e-11)
    w = np.array([2.0, 2.0, 1.5, 0.3, 0.0, 1.0])
    rho = torch.zeros(b.N, dtype=torch.float64, device=ctx().device)
    kb.density_accumulate(to_dev(psi), w, rho)
    ref = sum(w[i] * b.ifft_normalization ** 2 * np.abs(b.ifft_kpt(blk.kpt, psi[i], False)) ** 2 for i in range(6))
    np.testing.assert_allclose(rho.cpu().numpy(), ref, atol=1e-12 * ref.max())


@pytest.mark.parametrize("backend", [2, 4])   # 2: integer products on CUDA cores, 4: wgmma s8 on the tensor cores (TMA-fed, i8tc2.cu)
@pytest.mark.parametrize("shape", [(3000, 7, 5), (70000, 20, 9), (140000, 150, 130)])
def test_i8_emulated_gemm_matches_fp64(shape, backend):
    from gpu_common import ctx
    K, m, n = shape
    c = ctx()
    g = torch.Generator(device="cpu").manual_seed(1)
    decay = torch.exp(-torch.linspace(0, 30, K, dtype=torch.float64))
    A = (torch.view_as_complex(torch.randn(m, K, 2, generator=g, dtype=torch.float64)) * decay).to(c.device)
    B = (torch.view_as_complex(torch.randn(n, K, 2, generator=g, dtype=torch.float64)) * decay.sqrt()).to(c.device)
    ref = torch.zeros((n, m), dtype=torch.complex128, device=c.device)
    c.set_option("gemm_backend", 0)                  # reference: the FP64 DMMA kernels
    c.zgemm("C", A, B, ref)
    c.set_option("gemm_backend", backend)
    c.set_option("i8_min_rows", 1024)
    try:
        C = torch.zeros_like(ref)
        c.zgemm("C", A, B, C)
    finally:
        c.set_option("gemm_backend", 0)
        c.set_option("i8_min_rows", 32768)
    assert (C - ref).abs().max().item() < 1e-14 * ref.abs().max().item() * K ** 0.5
    if backend == 4:
        # update type on the tensor cores (A as the MN-major operand, its column scales folded into S): X = A S (+ X0)
        S = torch.view_as_complex(torch.randn(n, m, 2, generator=g, dtype=torch.float64)).to(c.device)
        X0 = torch.view_as_complex(torch.randn(n, K, 2, generator=g, dtype=torch.float64)).to(c.device)
        want = torch.zeros_like(X0)
        c.set_option("gemm_backend", 0)
        c.zgemm("N", A, S, want)
        c.set_option("gemm_backend", 4)
        c.set_option("i8_min_rows", 1024)
        try:
            X = torch.zeros_like(X0)
            c.zgemm("N", A, S, X)
            Xa = X0.clone()
            c.zgemm("N", A, S, Xa, -1.0, 1.0)
        finally:
            c.set_option("gemm_backend", 0)
            c.set_option("i8_min_rows", 32768)
        scale = (A.abs().max(dim=1).values[None, :] * S.abs()).sum(dim=1).max().item()      # sum_k |A[:,k]|max |S[k,j]|
        assert (X - want).abs().max().item() < 1e-14 * scale
        assert (Xa - X0 + want).abs().max().item() < 1e-14 * scale
    if backend == 2 and m * K < 3_000_000:
        # update type: X (K x n) = A (K x m) S (m x n), and the accumulating form, through the reference pipeline
        S = torch.view_as_complex(torch.randn(n, m, 2, generator=g, dtype=torch.float64)).to(c.device)
        X0 = torch.view_as_complex(torch.randn(n, K, 2, generator=g, dtype=torch.float64)).to(c.device)
        want = torch.zeros_like(X0)
        c.zgemm("N", A, S, want)
        c.set_option("gemm_backend", 2)
        try:
            X = torch.zeros_like(X0)
            c.zgemm("N", A, S, X)
            Xa = X0.clone()
            c.zgemm("N", A, S, Xa, 1.0, 1.0)
        finally:
            c.set_option("gemm_backend", 0)
        scale = (A.abs().max(dim=0).values[:, None] * S.abs().max()).max().item() * m
        assert (X - want).abs().max().item() < 1e-14 * scale
        assert (Xa - X0 - want).abs().max().item() < 1e-14 * scale


@pytest.mark.parametrize("backend,small", [(0, 1), (1, 0), (0, 0)])
def test_lobpcg_matches_oracle(si, backend, small):
    # small = 1: fused small-matrix kernels (lobpcg_small.cuh, the default for <= 32 bands);
    # small = 0: tensor-core GEMM + cuSOLVER sequence of the large path on the same problem
    from gpu_common import to_dev, ctx
    from oracle import lobpcg as olob
    ctx().set_option("gemm_backend", backend)
    ctx().set_option("small_dense", small)
    try:
        blk, kb = si["blk"], si["kb"]
        rng = np.random.default_rng(5)
        X0 = rng.standard_normal((blk.kpt.n_G, 8)) + 1j * rng.standard_normal((blk.kpt.n_G, 8))
        ref = olob.lobpcg(blk, X0.copy(), olob.PreconditionerTPA(blk.kin), tol=1e-9, maxiter=200)
        X = to_dev(X0.T)
        res = kb.lobpcg(X, tol=1e-9, maxiter=200)
        assert res["converged"] and ref["converged"]
        np.testing.assert_allclose(res["λ"], ref["λ"], atol=1e-8)
        assert abs(res["n_iter"] - ref["n_iter"]) <= max(3, ref["n_iter"] // 5)
        # residual check with the device operator itself
        HX = kb.apply_h(X)
        r = HX - torch.from_numpy(res["λ"]).to(X.device)[:, None] * X
        assert r.norm(dim=1).max().item() < 1e-8
        G = X.conj() @ X.T
        assert (G - torch.eye(8, dtype=G.dtype, device=G.device)).abs().max().item() < 1e-12
        # partial convergence / locking path: only 4 of 7 bands must converge (AdaptiveBands usage)
        X = to_dev(X0.T[:7])
        res2 = kb.lobpcg(X, tol=1e-7, maxiter=100, n_conv_check=4)
        np.testing.assert_allclose(res2["λ"][:4], ref["λ"][:4], atol=1e-6)
        # a rank-deficient start block (two identical columns) goes through the shifted safe_cholesky retries
        Xd = X0.T[:6].copy()
        Xd[4] = Xd[1]
        X = to_dev(Xd)
        res3 = kb.lobpcg(X, tol=1e-8, maxiter=200)
        assert res3["converged"]
        np.testing.assert_allclose(res3["λ"], ref["λ"][:6], atol=1e-7)
    finally:
        ctx().set_option("gemm_backend", 0)
        ctx().set_option("small_dense", 1)


def test_lobpcg_multi_matches_single_solves_and_oracle():
    """dftk_b200_lobpcg_multi (all k-blocks of a rank in lockstep, one launch per operation for all of them) against
    (a) the same blocks solved one at a time and (b) the oracle: same eigenvalues, same iteration counts per block.
    Blocks of different size (different k -> different n_pw), different convergence speed, partial convergence."""
    import dftk_b200
    from dftk_b200.device import lobpcg_multi
    from gpu_common import silicon_setup, device_blocks, to_dev, ctx
    from oracle import lobpcg as olob
    ks = [(0.1, -0.2, 0.3), (0.0, 0.0, 0.0), (0.5, 0.0, 0.0), (0.25, 0.25, -0.125), (0.5, 0.5, 0.5)]
    m, b, t, rho, ham = silicon_setup(Ecut=12, fft_size=(24, 24, 24), kcoords=ks, kweights=[0.2] * 5)
    grid, kbs = device_blocks(b, ham)
    assert len({kb.n_pw for kb in kbs}) > 1
    rng = np.random.default_rng(11)
    nb = 7
    X0 = [rng.standard_normal((blk.kpt.n_G, nb)) + 1j * rng.standard_normal((blk.kpt.n_G, nb)) for blk in ham]
    c = ctx()
    c.launch_count(reset=True)
    single = [kb.lobpcg(to_dev(x.T), tol=1e-8, maxiter=100, n_conv_check=5) for kb, x in zip(kbs, X0)]
    launches_single = c.launch_count(reset=True)
    c.sync_count(reset=True)
    Xs = [to_dev(x.T) for x in X0]
    multi = lobpcg_multi(kbs, Xs, tol=1e-8, maxiter=100, n_conv_check=5)
    launches_multi, rounds = c.launch_count(reset=True), c.sync_count()
    for blk, kb, x0, rs, rm, X in zip(ham, kbs, X0, single, multi, Xs):
        ref = olob.lobpcg(blk, x0.copy(), olob.PreconditionerTPA(blk.kin), tol=1e-8, maxiter=100, n_conv_check=5)
        assert rm["converged"] and rs["converged"] and ref["converged"]
        np.testing.assert_allclose(rm["λ"][:5], ref["λ"][:5], atol=1e-7)
        np.testing.assert_allclose(rm["λ"], rs["λ"], atol=1e-11)
        assert rm["n_iter"] == rs["n_iter"] and rm["n_matvec"] == rs["n_matvec"]
        assert abs(rm["n_iter"] - ref["n_iter"]) <= max(3, ref["n_iter"] // 5)
        r = kb.apply_h(X) - torch.from_numpy(rm["λ"]).to(X.device)[:, None] * X
        assert r.norm(dim=1)[:5].max().item() < 1e-8
        G = X.conj() @ X.T
        assert (G - torch.eye(nb, dtype=G.dtype, device=G.device)).abs().max().item() < 1e-12
    # the point of the exercise: far fewer launches than block-by-block, one synchronisation per round for all blocks
    assert launches_multi < 0.5 * launches_single, (launches_multi, launches_single)
    assert rounds > 0


def test_lobpcg_svd_fallback_recovers_rank_deficient_block(si):
    """ortho! falls back to an SVD when safe_cholesky gives up (lobpcg_hyper_impl.jl:226-231; the reference recovers
    through X <- U V').  With finite data five shifted factorisations practically never all fail, so the test forces the
    branch (option force_svd_fallback) on a start block with an exactly vanishing and a duplicated column: the fallback
    must hand back an orthonormal block and the solve must converge to the oracle's eigenvalues (both LOBPCG paths)."""
    from gpu_common import to_dev, ctx
    from oracle import lobpcg as olob
    blk, kb = si["blk"], si["kb"]
    rng = np.random.default_rng(9)
    X0 = rng.standard_normal((blk.kpt.n_G, 6)) + 1j * rng.standard_normal((blk.kpt.n_G, 6))
    ref = olob.lobpcg(blk, X0.copy(), olob.PreconditionerTPA(blk.kin), tol=1e-8, maxiter=200)
    for small in (1, 0):
        ctx().set_option("small_dense", small)
        try:
            Xd = X0.T.copy()
            Xd[2] = Xd[0]            # duplicated column
            Xd[3] = 0.0              # an exactly vanishing column
            ctx().set_option("force_svd_fallback", 2)
            res = kb.lobpcg(to_dev(Xd), tol=1e-8, maxiter=300)
            assert res["converged"]
            np.testing.assert_allclose(res["λ"], ref["λ"], atol=1e-7)
        finally:
            ctx().set_option("small_dense", 1)
            ctx().set_option("force_svd_fallback", 0)


def test_kblock_trim_frees_scratch_and_calls_regrow_it(si):
    """dftk_b200_kblock_trim: the scratch of earlier calls (solver workspaces, FFT intermediates) is returned to the device;
    the operator data stays, so the same calls give the same results afterwards."""
    from gpu_common import to_dev
    blk, kb = si["blk"], si["kb"]
    rng = np.random.default_rng(11)
    X0 = rng.standard_normal((blk.kpt.n_G, 6)) + 1j * rng.standard_normal((blk.kpt.n_G, 6))
    psi = to_dev(X0.T)
    h0 = kb.apply_h(psi).clone()
    r0 = kb.lobpcg(to_dev(X0.T), tol=1e-9, maxiter=200)
    free_before = kb.ctx.mem_info()[0]
    kb.trim()
    assert kb.ctx.mem_info()[0] >= free_before
    assert (kb.apply_h(psi) - h0).abs().max().item() <= 1e-13 * h0.abs().max().item()
    r1 = kb.lobpcg(to_dev(X0.T), tol=1e-9, maxiter=200)
    assert r0["converged"] and r1["converged"]
    np.testing.assert_allclose(r1["λ"], r0["λ"], atol=1e-9)


@pytest.mark.parametrize("fft_size,Ecut", [((40, 45, 48), 30), ((32, 27, 36), 14), ((33, 40, 21), 10),
                                           ((75, 64, 60), 60)])
def test_fft_engines_agree_with_oracle(fft_size, Ecut):
    """Register two-pass engine (default) and the generic Stockham engine against the oracle on mixed sizes
    (33 and 21 have no factor pair -> those axes fall back to the generic engine inside the same pipeline)."""
    import dftk_b200
    from gpu_common import ctx, to_dev, rand_psi
    from oracle.basis import Element, Model, PlaneWaveBasis
    from silicon import LATTICE, POSITIONS
    m = Model(LATTICE, [Element("Si")] * 2, POSITIONS, symmetries=False)
    b = PlaneWaveBasis(m, Ecut, fft_size=fft_size, kcoords=[[0.25, -0.1, 0.4]], kweights=[1.0])
    kpt = b.kpoints[0]
    rng = np.random.default_rng(7)
    V = rng.standard_normal(b.N)
    kin = rng.random(kpt.n_G)
    psi = rand_psi(kpt.n_G, 4, seed=8)
    ref = np.stack([b.fft_kpt(kpt, b.ifft_kpt(kpt, p, False) * V / b.N, False) + kin * p for p in psi])
    refc = np.stack([b.ifft_kpt(kpt, p) for p in psi])
    w = np.array([1.0, 0.5, 2.0, 0.25])
    refr = sum(w[i] * b.ifft_normalization ** 2 * np.abs(b.ifft_kpt(kpt, psi[i], False)) ** 2 for i in range(4))
    for engine in (0, 1):
        ctx().set_option("fft_engine", engine)
        try:
            grid = dftk_b200.FFTGrid(ctx(), fft_size, m.unit_cell_volume)
            kb = dftk_b200.KBlock(grid, kpt.mapping, kin=kin)
            kb.set_potential(to_dev(V))
            d = to_dev(psi)
            np.testing.assert_allclose(kb.apply_terms(d, 3).cpu().numpy(), ref, atol=1e-12 * np.abs(ref).max())
            cube = kb.sphere_to_real(d)
            np.testing.assert_allclose(cube.cpu().numpy(), refc, atol=1e-12 * np.abs(refc).max())
            np.testing.assert_allclose(kb.real_to_sphere(cube).cpu().numpy(), psi, atol=1e-12)
            rho = torch.zeros(b.N, dtype=torch.float64, device=ctx().device)
            kb.density_accumulate(d, w, rho)
            np.testing.assert_allclose(rho.cpu().numpy(), refr, atol=1e-12 * refr.max())
        finally:
            ctx().set_option("fft_engine", 0)


def _full_size_checks(rep, n, n_pw):
    """Si rep x rep x rep supercell, Gamma, Ecut 30 Ha on an n^3 grid: size-independent properties instead of an oracle
    run -- round trip, linearity, Hermiticity <phi|H psi> = <H phi|psi>, Parseval, density normalisation -- and
    apply_terms(psi, 3) and sphere_to_real of three bands against numpy.fft (which test_fft_reference.py ties to the
    direct DFT)."""
    import dftk_b200
    from gpu_common import ctx
    c = ctx()
    dev = c.device
    A = 10.26 / 2
    lat = rep * np.array([[0, A, A], [A, 0, A], [A, A, 0]])
    recip = 2 * np.pi * np.linalg.inv(lat.T)
    g1 = torch.as_tensor(np.array(list(range(0, (n + 1) // 2)) + list(range(-(n // 2), 0))), device=dev, dtype=torch.float64)
    Z, Y, X = torch.meshgrid(g1, g1, g1, indexing="ij")
    G = torch.stack([X.reshape(-1), Y.reshape(-1), Z.reshape(-1)], 1)
    p = G @ torch.as_tensor(recip.T, device=dev)
    kin_all = (p * p).sum(1) / 2
    del G, p, X, Y, Z
    mapping = torch.nonzero(kin_all <= 30.0).reshape(-1)
    assert mapping.numel() == n_pw
    kin = kin_all[mapping].contiguous()
    del kin_all
    vol = abs(np.linalg.det(lat))
    grid = dftk_b200.FFTGrid(c, (n, n, n), vol)
    kb = dftk_b200.KBlock(grid, mapping.cpu().numpy(), kin=kin)
    V = torch.cos(torch.arange(n ** 3, device=dev, dtype=torch.float64) * 1e-3) - 0.3
    kb.set_potential(V)
    gen = torch.Generator(device=dev).manual_seed(1)
    psi = torch.view_as_complex(torch.randn(6, mapping.numel(), 2, generator=gen, device=dev, dtype=torch.float64))
    psi = psi / psi.norm(dim=1, keepdim=True)
    cube = kb.sphere_to_real(psi)
    # Parseval: sum |psi(r)|^2 dvol = 1
    assert (cube.abs().pow(2).sum(dim=1) * (vol / n ** 3) - 1).abs().max().item() < 1e-12
    assert (kb.real_to_sphere(cube) - psi).abs().max().item() < 1e-13
    del cube
    H = kb.apply_h(psi)
    a, b = 0.3 - 1.2j, -0.7 + 0.4j
    Hlin = kb.apply_h((a * psi[0] + b * psi[1])[None, :].contiguous())[0]
    assert (Hlin - (a * H[0] + b * H[1])).abs().max().item() < 1e-12 * H.abs().max().item()
    Gm = psi.conj() @ H.T
    assert (Gm - Gm.conj().T).abs().max().item() < 1e-12 * Gm.abs().max().item()
    rho = torch.zeros(n ** 3, dtype=torch.float64, device=dev)
    kb.density_accumulate(psi, np.full(6, 2.0), rho)
    assert abs(rho.sum().item() * (vol / n ** 3) - 12.0) < 1e-10
    assert rho.min().item() >= 0.0
    del rho, H
    # three bands against numpy.fft
    mp, Vn, kn = mapping.cpu().numpy(), V.cpu().numpy().reshape(n, n, n), kin.cpu().numpy()
    ps = psi[:3].contiguous()
    hp = kb.apply_terms(ps, 3).cpu().numpy()
    cube = kb.sphere_to_real(ps).cpu().numpy()
    ps = ps.cpu().numpy()
    for i in range(3):
        c3 = np.zeros(n ** 3, dtype=complex)
        c3[mp] = ps[i]
        r = np.fft.ifftn(c3.reshape(n, n, n))
        ref = r.reshape(-1) * (n ** 3 / np.sqrt(vol))
        assert np.abs(cube[i] - ref).max() <= 1e-13 * np.abs(ref).max()
        ref = np.fft.fftn(r * Vn).reshape(-1)[mp] + kn * ps[i]
        assert np.abs(hp[i] - ref).max() <= 1e-13 * np.abs(ref).max()


def test_full_size_properties_192():
    """BASELINE full-size grid (192^3, the C3 cell: Si 5x5x5 supercell)."""
    _full_size_checks(5, 192, 264859)                              # SURVEY §8 table, config C3


def test_full_size_properties_150():
    """The benchmark cell's grid (150^3, Si 4x4x4 supercell, the n_pw of bench.py's flagship workload)."""
    _full_size_checks(4, 150, 135491)


def test_against_committed_golden_fixture():
    """Committed vectors (tests/golden/si_block_fixture.npz, made by tests/golden/make_fixtures.py): the CUDA
    path must reproduce the stored Hψ, eigenvalues and density from the stored operator data alone."""
    import os
    import dftk_b200
    from gpu_common import ctx, to_dev
    f = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "si_block_fixture.npz"))
    grid = dftk_b200.FFTGrid(ctx(), tuple(int(x) for x in f["fft_size"]), float(f["volume"]))
    kb = dftk_b200.KBlock(grid, f["mapping"], kin=f["kin"], P=to_dev(f["P"].T), D=f["D"])
    kb.set_potential(to_dev(f["V"]))
    h = kb.apply_h(to_dev(f["psi"])).cpu().numpy()
    np.testing.assert_allclose(h, f["hpsi"], atol=1e-12 * np.abs(f["hpsi"]).max())
    X = to_dev(f["psi"])
    res = kb.lobpcg(X, tol=1e-10, maxiter=200)
    np.testing.assert_allclose(res["λ"], f["eigenvalues"], atol=1e-9)
    rho = torch.zeros(grid.N, dtype=torch.float64, device=ctx().device)
    kb.density_accumulate(X, f["occ"], rho)
    np.testing.assert_allclose(rho.cpu().numpy(), f["rho"], atol=1e-9 * f["rho"].max())


def test_host_buffer_pipeline_many_bands(si):
    """End-to-end path of the C ABI (host psi/hpsi): more bands than one staging chunk (128) so that the
    double-buffered H2D / compute / D2H pipeline wraps around several times."""
    from gpu_common import rand_psi
    from dftk_b200._lib import check
    from dftk_b200.device import _ptr
    blk, kb = si["blk"], si["kb"]
    nb = 300
    psi = rand_psi(blk.kpt.n_G, nb, seed=11)
    psi_pin = torch.from_numpy(psi).pin_memory()
    out_pin = torch.empty_like(psi_pin).pin_memory()
    check(kb.ctx.L.dftk_b200_apply_h(kb.h, _ptr(psi_pin), _ptr(out_pin), nb), kb.ctx.h)
    ref = blk.matmul(psi.T).T
    np.testing.assert_allclose(out_pin.numpy(), ref, atol=1e-12 * np.abs(ref).max())
    # device-resident result of the same call must be identical (same kernels, same order)
    dev = kb.apply_h(torch.from_numpy(psi).to(kb.ctx.device)).cpu().numpy()
    np.testing.assert_allclose(out_pin.numpy(), dev, atol=1e-13 * np.abs(ref).max())


def test_unsorted_mapping_falls_back(si):
    """construct_from_equivalent_kpt (src/Kpoint.jl:44-56) yields mappings that are not ascending: the library
    must still be exact (such k-blocks are routed to the generic FFT engine)."""
    import dftk_b200
    from gpu_common import to_dev, rand_psi, ctx
    b, blk = si["b"], si["blk"]
    kpt = blk.kpt
    rng = np.random.default_rng(12)
    perm = rng.permutation(kpt.n_G)
    grid = dftk_b200.FFTGrid(ctx(), b.fft_size, b.model.unit_cell_volume)
    kb = dftk_b200.KBlock(grid, kpt.mapping[perm], kin=blk.kin[perm])
    kb.set_potential(to_dev(blk.Vtot))
    psi = rand_psi(kpt.n_G, 3, seed=13)
    ref = blk.local_apply(psi.T).T + blk.kin[None, :] * psi
    out = kb.apply_terms(to_dev(psi[:, perm]), 3).cpu().numpy()
    np.testing.assert_allclose(out, ref[:, perm], atol=1e-12 * np.abs(ref).max())


@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("funs", [("lda_x", "lda_c_vwn"), ("lda_x", "lda_c_pw"), ("gga_x_pbe", "gga_c_pbe")])
def test_xc_kernel_matches_oracle(n_spin, funs):
    from dftk_b200 import xc as pxc
    from gpu_common import ctx, to_dev
    from oracle import xc as oxc
    rng = np.random.default_rng(21)
    N = 5000
    rho = rng.random((n_spin, N)) * 0.4 + 1e-6
    rho[:, :5] = 0.0
    gga = funs[0].startswith("gga")
    sigma = None
    if gga:
        sigma = rng.random((1 if n_spin == 1 else 3, N)) * 0.02
        if n_spin == 2:
            sigma[1] = np.sqrt(sigma[0] * sigma[2]) * rng.uniform(-1, 1, N)
    e, vr, vs = pxc.evaluate(ctx(), list(funs), to_dev(rho), None if sigma is None else to_dev(sigma))
    ref = oxc.evaluate(list(funs), rho, sigma)
    np.testing.assert_allclose(e.cpu().numpy(), ref["e"], rtol=1e-12, atol=1e-16)
    np.testing.assert_allclose(vr.cpu().numpy(), ref["Vrho"], rtol=1e-11, atol=1e-14)
    if gga:
        np.testing.assert_allclose(vs.cpu().numpy(), ref["Vsigma"], rtol=1e-10, atol=1e-13)


def test_symmetrize_kernel_matches_oracle():
    """dftk_b200_symmetrize_fourier on aluminium fcc (192 operations, half of them with fractional translations)."""
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle.scf import symmetrize_rho as osym
    a = 7.65339
    pos = [[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]]
    Al = dftk.ElementPsp("Al", functional="pbe")
    model = dftk.model_DFT(a * np.eye(3), [Al] * 4, pos, functionals=dftk.PBE(), temperature=0.01)
    basis = dftk.PlaneWaveBasis(model, Ecut=5, kgrid=(2, 2, 2))
    om = Model(a * np.eye(3), [Element("Al", functional="pbe")] * 4, pos, functionals=("gga_x_pbe", "gga_c_pbe"),
               temperature=0.01)
    ob = OBasis(om, 5, kgrid=(2, 2, 2))
    assert len(basis.symmetries) == len(ob.symmetries) == 192 and basis.fft_size == ob.fft_size
    rng = np.random.default_rng(3)
    rho = rng.random((1, ob.N))
    out = dftk.symmetrize_rho(basis, torch.from_numpy(rho).to(basis.architecture.device)).cpu().numpy()
    np.testing.assert_allclose(out, osym(ob, rho), atol=1e-13)
