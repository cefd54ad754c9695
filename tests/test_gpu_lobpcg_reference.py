"""The device LOBPCG solvers (KBlock.lobpcg on the batched small path and on the tensor-core + cuSOLVER path,
lobpcg_multi in lockstep) against a dense diagonalisation of the same Hamiltonian (tests/lobpcg_reference.py), at the
band-count, locking and spectrum edges.  Run on an H100: -m gpu."""
import numpy as np
import pytest
import torch

import lobpcg_reference as lr

pytestmark = pytest.mark.gpu

TOL = 1e-9
DEFAULTS = dict(gemm_backend=0, small_dense=1, batch_pipeline=0)
_GRIDS = {}
_KBS = {}


def _grid(fft_size):
    import dftk_b200
    from gpu_common import ctx
    if fft_size not in _GRIDS:
        _GRIDS[fft_size] = dftk_b200.FFTGrid(ctx(), fft_size, 270.0)
    return _GRIDS[fft_size]


def kblock(name, nb, seed=0):
    """Device k-block of CASES[name](nb, seed); blocks of one FFT size share a grid, as the blocks of a basis do."""
    import dftk_b200
    from gpu_common import to_dev
    key = (name, nb if name.startswith("tight") else 0, seed)
    if key not in _KBS:
        case = lr.problem(name, nb, seed)[0]
        P = None if case.P is None else to_dev(case.P.T)
        kb = dftk_b200.KBlock(_grid(tuple(case.fft_size)), case.mapping, kin=case.kin, P=P, D=case.D)
        if case.V is not None:
            kb.set_potential(to_dev(case.V))
        _KBS[key] = kb
    return _KBS[key]


class options:
    """Set context options for a block of code and put the defaults back afterwards."""

    def __init__(self, **kw):
        self.kw = kw

    def __enter__(self):
        from gpu_common import ctx
        for k, v in self.kw.items():
            ctx().set_option(k, v)

    def __exit__(self, *exc):
        from gpu_common import ctx
        for k in self.kw:
            ctx().set_option(k, DEFAULTS[k])
        return False


def _host(X):
    return X.cpu().numpy().T.copy()


def n_conv_check_for(name, nb, which):
    if name == "si-gamma" and nb >= 31:
        return nb - 6                       # the highest bands sit in a dense part of the spectrum: unconverged extra bands
    return {0: nb, 1: max(1, nb // 2), 2: 1}[which]


@pytest.mark.parametrize("name", list(lr.CASES))
def test_apply_h_is_the_dense_operator(name):
    """Localises a failure below: H X from the device equals the dense H times X."""
    from gpu_common import to_dev
    nb = 5
    case, H, spec = lr.problem(name, nb)
    X0 = lr.start_block("random", spec, nb)[0]
    got = _host(kblock(name, nb).apply_h(to_dev(X0.T)))
    ref = H @ X0
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()


SINGLE_NB = (1, 2, 3, 8, 31, 32, 33, 40, 64)


def _single_params():
    """One row per (case, band count), on both paths up to 32 bands.  The start kind advances with the case and with the
    band count, so every band count meets every start kind (twice and more over the nine cases) and every case meets every
    kind; n_conv_check (nb, nb/2, 1), miniter (0 for the starts with exact columns, else 1 or 3) and the unpreconditioned
    runs advance with other strides."""
    out = []
    for ci, name in enumerate(lr.CASES):
        for ni, nb in enumerate(SINGLE_NB):
            if nb == 64 and not name.startswith("si"):
                continue
            kind = lr.START_KINDS[(ci + ni) % 4]
            if kind == "exact-high-first" and (nb == 1 or (name == "si-gamma" and nb >= 31)):
                kind = "random"     # one column: just an exact start; Gamma: `converged` is taken over the sorted columns
            prec = not ((ci + ni) % 3 == 2 and name in ("si-k", "tight+1", "tight+5"))
            which = 0 if kind == "exact-high-first" else (ci + 2 * ni) % 3
            miniter = 0 if kind != "random" else (1, 3)[(ci + ni // 4) % 2]
            for small in ((1, 0) if nb <= 32 else (0,)):
                backend = 0 if small else (ci + ni) % 2
                out.append((name, nb, kind, prec, which, miniter, small, backend))
    # 32 bands from a random start, all of them to convergence: the small path then runs its 96-column Rayleigh-Ritz and two
    # full 16-column chunks for many iterations
    for name, prec, miniter in (("si-k", True, 1), ("diag-degenerate", True, 3), ("tight+5", False, 1)):
        out += [(name, 32, "random", prec, 0, miniter, small, 0) for small in (1, 0)]
    return [pytest.param(*r, id="{}-{}-{}-prec{:d}-ncc{}-min{}-small{}-be{}".format(*r)) for r in out]


def test_single_solve_table_covers_the_pairings():
    rows = [p.values for p in _single_params()]
    for nb in SINGLE_NB[1:-1]:            # 64 bands run on the two silicon blocks only
        assert {r[2] for r in rows if r[1] == nb} == set(lr.START_KINDS), nb
    for name in lr.CASES:
        assert {r[2] for r in rows if r[0] == name} == set(lr.START_KINDS), name
    assert {r[5] for r in rows} == {0, 1, 3} and {r[4] for r in rows} == {0, 1, 2}
    assert {(r[3], r[6]) for r in rows} == {(True, 1), (True, 0), (False, 1), (False, 0)}
    assert {r[7] for r in rows if r[6] == 0} == {0, 1}
    assert any(r[1] == 32 and r[2] == "random" and r[6] == 1 and r[4] == 0 for r in rows)


@pytest.mark.parametrize("name,nb,kind,prec,which,miniter,small,backend", _single_params())
def test_kblock_lobpcg_against_dense_diagonalisation(name, nb, kind, prec, which, miniter, small, backend):
    """KBlock.lobpcg through check_solution, on the small path (small_dense = 1, <= 32 bands) and on the large one.
    A column locked before the last iteration reports a residual norm of exactly 0.0, as in the reference (the history
    is zero-initialised, lobpcg_hyper_impl.jl:367; an iteration writes the rows of its active columns only, :445; the
    result is the column of the last iteration, :336): check_solution asserts that and that the true residual of such a
    column is still below tol.  The iteration count is compared with the NumPy twin on the well-conditioned cases."""
    from gpu_common import to_dev
    from oracle import lobpcg as olob
    case, H, spec = lr.problem(name, nb)
    X0, expected, n_exact = lr.start_block(kind, spec, nb)
    ncc = n_conv_check_for(name, nb, which)
    kb = kblock(name, nb)
    X = to_dev(X0.T)
    with options(small_dense=small, gemm_backend=backend):
        # the 1e-6-split clusters of near-degenerate resolve at a pace that depends on rounding
        res = kb.lobpcg(X, tol=TOL, miniter=miniter, maxiter=600 if name == "near-degenerate" else 300, n_conv_check=ncc, prec=prec)
    Xh = _host(X)
    lr.check_solution(H, res, Xh, nb, ncc, TOL, spec=spec, expected=expected)
    assert res["converged"], (res["n_iter"], res["residual_norms"])
    if kind == "exact":
        assert res["n_iter"] == max(0, miniter) and res["n_matvec"] == nb
    if kind == "partly-exact" and res["n_iter"] > 0 and ncc == nb:
        assert np.all(res["residual_norms"][:n_exact] == 0.0)
        assert res["n_matvec"] <= nb + res["n_iter"] * (nb - n_exact)
    if kind == "exact-high-first" and nb > 1:
        lr.check_moved_column(H, res, Xh, spec, expected[-1])
    if name in lr.WELL_CONDITIONED and kind != "exact":
        ref = olob.lobpcg(lr.DenseOperator(H), X0.copy(), olob.PreconditionerTPA(case.kin) if prec else None, tol=TOL,
                          maxiter=300, miniter=miniter, n_conv_check=ncc)
        assert ref["converged"]
        assert abs(res["n_iter"] - ref["n_iter"]) <= max(3, ref["n_iter"] // 5), (res["n_iter"], ref["n_iter"])


@pytest.mark.parametrize("name,nb,small", [("si-k", 8, 1), ("si-k", 8, 0), ("wide-range", 40, 0), ("tight+1", 32, 1)])
@pytest.mark.parametrize("prec", [True, False])
def test_maxiter_reached_returns_a_consistent_unconverged_result(name, nb, small, prec):
    """maxiter = 3 at tol = 1e-12: no error, converged == False, and what is returned is still orthonormal, with lambda
    the Rayleigh quotients and the reported residuals the true ones (check_solution)."""
    from gpu_common import to_dev
    case, H, spec = lr.problem(name, nb)
    X0 = lr.start_block("random", spec, nb)[0]
    X = to_dev(X0.T)
    with options(small_dense=small):
        res = kblock(name, nb).lobpcg(X, tol=1e-12, maxiter=3, prec=prec)
    assert res["converged"] is False and res["n_iter"] == 3
    assert res["n_matvec"] == 4 * nb
    lr.check_solution(H, res, _host(X), nb, nb, 1e-12, spec=spec)          # reported residuals = true ones to 1e-6 relative
    assert np.all(res["residual_norms"] > 1e-12)


def test_int8_backend_against_dense_diagonalisation():
    """gemm_backend 4 at 40 bands: with i8_min_rows lowered to 2048 the Gram and update products of the large path and the
    projection run on the INT8 tensor cores (a silicon block of more than 2048 plane waves)."""
    from gpu_common import ctx, to_dev
    import dftk_b200
    nb = 40
    case, H, spec = lr.large_silicon_problem()
    assert H.shape[0] > 2048
    kb = dftk_b200.KBlock(_grid(tuple(case.fft_size)), case.mapping, kin=case.kin, P=to_dev(case.P.T), D=case.D)
    kb.set_potential(to_dev(case.V))
    X0, expected, _ = lr.start_block("random", spec, nb)
    X = to_dev(X0.T)
    ctx().set_option("gemm_backend", 4)
    ctx().set_option("i8_min_rows", 2048)
    try:
        res = kb.lobpcg(X, tol=TOL, maxiter=300)
    finally:
        ctx().set_option("gemm_backend", 0)
        ctx().set_option("i8_min_rows", 32768)
    lr.check_solution(H, res, _host(X), nb, nb, TOL, spec=spec, expected=expected)
    assert res["converged"]


BATCHES = {
    # (case, seed) per block.  One FFT grid (12^3), different n_pw: the blocks of a basis, whose local terms go through
    # one fused multi-block FFT launch; every block qualifies for the two-group scheduler of batch_pipeline = 1
    "one": [("si-k", 0)],
    "two": [("tight+5", 0), ("diag-degenerate", 0)],
    "nine": [("diag-degenerate", 0), ("tight+1", 0), ("near-degenerate", 0), ("tight+5", 0), ("many-projectors-96", 0),
             ("diag-degenerate", 1), ("near-degenerate", 1), ("many-projectors-96", 1), ("tight+5", 1)],
    # 97 projectors: that block's nonlocal term leaves the fused projection, and the batch stays in one group
    "nine-97": [("diag-degenerate", 0), ("tight+1", 0), ("near-degenerate", 0), ("tight+5", 0), ("many-projectors-97", 0),
                ("diag-degenerate", 1), ("near-degenerate", 1), ("many-projectors-96", 1), ("tight+5", 1)],
    # extra: three FFT grids in one call (the local term is then applied block by block)
    "nine-mixed-grids": [("si-gamma", 0), ("si-k", 0), ("diag-degenerate", 0), ("near-degenerate", 0), ("wide-range", 0),
                         ("tight+1", 0), ("tight+5", 0), ("many-projectors-96", 0), ("many-projectors-97", 0)],
}


@pytest.mark.parametrize("batch,nb,pipeline", [("one", 7, 0), ("two", 32, 0), ("two", 2, 1), ("two", 1, 0),
                                               ("nine", 7, 0), ("nine", 7, 1), ("nine", 31, 1), ("nine", 32, 0), ("nine", 2, 1),
                                               ("nine-97", 8, 0), ("nine-97", 8, 1),
                                               ("nine-mixed-grids", 7, 0), ("nine-mixed-grids", 7, 1)])
def test_lobpcg_multi_against_dense_diagonalisation_and_single_solves(batch, nb, pipeline):
    """lobpcg_multi: blocks of different n_pw in one call, one of them started from its exact eigenvectors (it finishes at
    round 0 while the others run on), one from a partly exact block and one from a block whose first column locks at once
    and must be moved by the final sort.  Every block goes through check_solution and is identical to KBlock.lobpcg on the
    same input: lambda to 1e-11, equal n_iter and n_matvec.  Only the batch over three FFT grids is compared within
    max(3, 20 %) iterations instead: there the local term is applied block by block, a single solve goes through the
    batched kernel, the two round differently, and inside degenerate clusters the count follows the rounding."""
    from dftk_b200.device import lobpcg_multi
    from gpu_common import to_dev
    blocks = BATCHES[batch]
    one_grid = len({tuple(lr.problem(n_, nb, s_)[0].fft_size) for n_, s_ in blocks}) == 1
    assert one_grid == (batch != "nine-mixed-grids")
    kinds = ["random"] * len(blocks)
    if len(blocks) > 1:
        kinds[1] = "exact"
    if len(blocks) > 2:
        kinds[3] = "partly-exact"
        kinds[5] = "exact-high-first"
    probs, starts, kbs = [], [], []
    for (name, seed), kind in zip(blocks, kinds):
        case, H, spec = lr.problem(name, nb, seed)
        probs.append((H, spec))
        starts.append(lr.start_block(kind, spec, nb, seed))
        kbs.append(kblock(name, nb, seed))
    assert len(blocks) == 1 or len({kb.n_pw for kb in kbs}) > 1
    kw = dict(tol=TOL, miniter=0, maxiter=600, n_conv_check=nb)
    single = []
    for kb, st in zip(kbs, starts):
        X = to_dev(st[0].T)
        single.append(kb.lobpcg(X, **kw))
    Xs = [to_dev(st[0].T) for st in starts]
    with options(batch_pipeline=pipeline):
        multi = lobpcg_multi(kbs, Xs, **kw)
    for (name, _), (H, spec), st, rs, rm, X, kind in zip(blocks, probs, starts, single, multi, Xs, kinds):
        Xh = _host(X)
        lr.check_solution(H, rm, Xh, nb, nb, TOL, spec=spec, expected=st[1])
        assert rm["converged"] and rs["converged"]
        if kind == "exact-high-first" and nb > 1:
            lr.check_moved_column(H, rm, Xh, spec, st[1][-1])
        np.testing.assert_allclose(rm["λ"], rs["λ"], rtol=0, atol=1e-11 * max(1.0, spec.norm))
        if one_grid:
            assert rm["n_iter"] == rs["n_iter"] and rm["n_matvec"] == rs["n_matvec"], (name, rm["n_iter"], rs["n_iter"])
        else:
            assert abs(rm["n_iter"] - rs["n_iter"]) <= max(3, rs["n_iter"] // 5), (name, rm["n_iter"], rs["n_iter"])
        if kind == "exact":
            assert rm["n_iter"] == 0 and rm["n_matvec"] == nb
    assert len({r["n_iter"] for r in multi}) > 1 or len(blocks) == 1


@pytest.mark.parametrize("small", [1, 0])
@pytest.mark.parametrize("nb,extra", [(7, 0), (7, -1), (33, 0), (33, -1)])
def test_too_small_problems_are_refused(nb, extra, small):
    """n_pw = 3 nb and 3 nb - 1: every entry point refuses on the host (init_solver) before any device work; X is left
    untouched.  The slab entry needs a communicator and refuses a one-rank context before it looks at the sizes."""
    import dftk_b200
    from dftk_b200.device import lobpcg_multi
    from gpu_common import to_dev
    n_pw = 3 * nb + extra
    fft_size = (12, 12, 12)
    rng = np.random.default_rng(0)
    kb = dftk_b200.KBlock(_grid(fft_size), lr.sphere_mapping(fft_size, n_pw), kin=1.0 + rng.random(n_pw))
    kb.set_potential(to_dev(np.zeros(12 ** 3)))
    X0 = rng.standard_normal((nb, n_pw)) + 1j * rng.standard_normal((nb, n_pw))
    X = to_dev(X0)
    with options(small_dense=small):
        with pytest.raises(dftk_b200.DftkB200Error, match="eigenproblem is too small"):
            kb.lobpcg(X, tol=TOL)
        with pytest.raises(dftk_b200.DftkB200Error, match="eigenproblem is too small"):
            lobpcg_multi([kblock("si-k", nb), kb], [to_dev(np.zeros((nb, kblock("si-k", nb).n_pw), dtype=complex)), X], tol=TOL)
        with pytest.raises(dftk_b200.DftkB200Error, match="no communicator"):
            kb.lobpcg_slab(X, tol=TOL)
    assert np.array_equal(X.cpu().numpy(), X0)
