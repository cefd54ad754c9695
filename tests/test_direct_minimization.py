"""CPU checks of direct_minimization: the host-side BackTracking and L-BFGS bookkeeping on small problems, and the NumPy
direct minimisation on the oracle against the oracle SCF (reference: test/scf_compare.jl)."""
import math
import numpy as np
import pytest

from dftk_b200.direct_minimization import (backtracking, LBFGSHistory, lbfgs_iteration, two_loop, _mod1,
                                           select_occupied_orbitals)
from silicon import LATTICE, POSITIONS, KCOORDS, KWEIGHTS


class EuclidOps:
    """Flat real vectors (one block), no manifold, identity preconditioner: the bookkeeping alone."""

    last_value = None

    def __init__(self):
        self.log = []

    def copy(self, a):
        return [t.copy() for t in a]

    def dot(self, a, b):
        self.log.append(("dot", id(a[0])))
        return float(sum(np.dot(x, y) for x, y in zip(a, b)))

    def axpy_dot(self, y, x, c, z=None):
        self.log.append(("axpy", id(x[0])))
        for yi, xi in zip(y, x):
            yi += c * xi
        return None if z is None else float(sum(np.dot(p, q) for p, q in zip(z, y)))

    def negate(self, s):
        for t in s:
            t *= -1

    def scaled(self, s, a):
        return [a * t for t in s]

    def add_scaled(self, x, s, a):
        return [xi + a * si for xi, si in zip(x, s)]

    def project(self, x, g):
        pass

    def retract(self, y):
        return [t.copy() for t in y]

    def precondprep(self, x):
        pass

    def ldiv(self, q):
        return [t.copy() for t in q]


def test_backtracking_accepts_the_full_step():
    phi = lambda a: -a + 0.1 * a * a
    a, v = backtracking(phi, 0.0, -1.0)
    assert a == 1.0 and v == phi(1.0)


def test_backtracking_quadratic_step_is_exact_on_a_parabola():
    calls = []

    def phi(a):
        calls.append(a)
        return (a - 0.3) ** 2
    a, v = backtracking(phi, 0.09, -0.6)
    # α_tmp = −dϕ0 / (2 (ϕ(1) − ϕ0 − dϕ0)) = 0.6 / (2 · 1.0) = 0.3: the minimiser, within [0.1, 0.5]
    assert calls[0] == 1.0
    assert a == pytest.approx(0.3, rel=1e-14) and v == pytest.approx(0.0, abs=1e-28)


def test_backtracking_cubic_step_is_exact_on_a_cubic():
    c = 2000.0
    calls = []

    def phi(a):
        calls.append(a)
        return -a + c * a ** 3
    a, _ = backtracking(phi, 0.0, -1.0)
    # first pass: quadratic step 1/(2·2000) clipped up to ρ_lo = 0.1; second pass: the cubic through (1, ϕ(1)) and
    # (0.1, ϕ(0.1)) is ϕ itself, whose minimiser is sqrt(1/(3c)), inside [0.01, 0.05]
    assert calls[:2] == [1.0, pytest.approx(0.1, rel=1e-15)]
    assert a == pytest.approx(math.sqrt(1 / (3 * c)), rel=1e-10)


def test_backtracking_halves_through_non_finite_values():
    a, v = backtracking(lambda a: math.inf if a > 0.2 else -a, 0.0, -1.0)
    assert a == 0.125 and v == -0.125


def test_ring_buffer_order_beyond_m():
    h = LBFGSHistory(m=10)
    h.pseudo_iteration = 13
    assert h.indices() == list(range(3, 13))
    assert [_mod1(i, 10) for i in h.indices()] == [3, 4, 5, 6, 7, 8, 9, 10, 1, 2]
    # the two-loop recursion visits the newest pair first on the way back and the oldest first on the way forward
    ops = EuclidOps()
    for i in range(1, 11):
        h.dx[i], h.dg[i], h.rho[i] = [np.full(3, float(i))], [np.full(3, 0.5 * i)], 1.0 / (1.5 * i * i)
    two_loop(ops, h, [np.ones(3)])
    back = [op for op in ops.log if op[0] == "axpy"][:10]
    fwd = [op for op in ops.log if op[0] == "axpy"][10:]
    assert [o[1] for o in back] == [id(h.dg[_mod1(i, 10)][0]) for i in range(12, 2, -1)]
    assert [o[1] for o in fwd] == [id(h.dx[_mod1(i, 10)][0]) for i in range(3, 13)]


def test_infinite_rho_is_skipped():
    h = LBFGSHistory(m=10)
    h.pseudo_iteration = 4
    keep = h.dx[4]
    assert not h.store([np.zeros(2)], [np.zeros(2)], 0.0)
    assert h.pseudo_iteration == 1 and h.dx[4] is keep
    h.pseudo_iteration = 4
    assert h.store([np.ones(2)], [np.ones(2)], 2.0)
    assert h.rho[4] == 0.5


def test_reset_on_an_ascent_direction():
    # a stored pair of negative curvature cancels the gradient: dϕ0 = 0 >= 0 resets to s = −P \ g
    ops = EuclidOps()
    h = LBFGSHistory(m=10)
    e1 = np.array([1.0, 0.0])
    h.dx[1], h.dg[1], h.rho[1] = [e1.copy()], [-e1], -1.0
    h.pseudo_iteration = 1
    f = lambda x: 0.5 * float(np.dot(x[0], x[0]))
    x = [e1.copy()]
    ops.last_value = f(x)

    def vg(y):
        ops.last_value = f(y)
        return f(y), [y[0].copy()]
    x_new, g_new, E, s = lbfgs_iteration(ops, h, x, [e1.copy()], f, vg)
    np.testing.assert_array_equal(s[0], -e1)
    np.testing.assert_array_equal(x_new[0], np.zeros(2))
    assert h.pseudo_iteration == 1 and h.rho[1] == 1.0 and E == 0.0


def test_lbfgs_minimises_a_quadratic():
    rng = np.random.default_rng(3)
    A = rng.standard_normal((12, 12))
    A = A @ A.T + 12 * np.eye(12)
    b = rng.standard_normal(12)
    f = lambda x: 0.5 * float(x[0] @ A @ x[0]) - float(b @ x[0])
    ops = EuclidOps()
    h = LBFGSHistory()

    def vg(y):
        ops.last_value = f(y)
        return f(y), [A @ y[0] - b]
    x = [np.zeros(12)]
    _, g = vg(x)
    for _ in range(40):
        x, g, _, _ = lbfgs_iteration(ops, h, x, g, f, vg)
        if g is None:
            break
    np.testing.assert_allclose(x[0], np.linalg.solve(A, b), atol=1e-9)
    assert h.pseudo_iteration == 40


def test_select_occupied_orbitals():
    import torch
    psi = [torch.arange(12.0).reshape(4, 3), torch.arange(8.0).reshape(4, 2)]
    occ = [np.array([2.0, 2.0, 0.0, 0.0]), np.array([2.0, 1e-3, 1e-9, 0.0])]
    out = select_occupied_orbitals(None, psi, occ, threshold=1e-6)
    assert [p.shape[0] for p in out["psi"]] == [2, 2]
    assert list(out["occupation"][1]) == [2.0, 1e-3]


class _StubBasis:
    """Just what direct_minimization inspects before it touches the device."""

    def __init__(self, temperature=0.0, nranks=1, comm_slab=None, hubbard=False):
        from types import SimpleNamespace
        self.model = SimpleNamespace(temperature=temperature)
        self.comm_kpts = SimpleNamespace(nranks=nranks, rank=0)
        self.comm_slab = comm_slab
        self._hub = object() if hubbard else None

    def term(self, name):
        return self._hub if name == "Hubbard" else None


def test_refusals_before_any_device_work():
    from dftk_b200 import direct_minimization
    with pytest.raises(ValueError):
        direct_minimization(_StubBasis(temperature=0.01))
    with pytest.raises(NotImplementedError, match="Direct minimization with MPI is not supported yet"):
        direct_minimization(_StubBasis(nranks=2))
    with pytest.raises(NotImplementedError):
        direct_minimization(_StubBasis(comm_slab=object()))
    with pytest.raises(NotImplementedError):
        direct_minimization(_StubBasis(hubbard=True))


# ---------------------------------------------------------------- the oracle minimisation against the oracle SCF
def _oracle_si(magnetic_moments=()):
    from oracle.basis import Element, Model, PlaneWaveBasis
    m = Model(LATTICE, [Element("Si")] * 2, POSITIONS, functionals=("lda_x", "lda_c_vwn"),
              magnetic_moments=magnetic_moments)
    return PlaneWaveBasis(m, 3, fft_size=(9, 9, 9), kcoords=KCOORDS, kweights=KWEIGHTS)


class NumpyOps:
    """The vector operations of the product's L-BFGS (DeviceOps) on host arrays, so that the product's host-side
    iteration can run on the oracle's energy without a GPU."""

    def __init__(self, kin, kweights, use_tpa=True):
        self.kin, self.kweights, self.use_tpa = kin, kweights, use_tpa
        self.mean_kin = None
        self.last_value = None

    def copy(self, a):
        return [t.copy() for t in a]

    def dot(self, a, b):
        return float(sum(np.real(np.vdot(x, y)) for x, y in zip(a, b)))

    def axpy_dot(self, y, x, c, z=None):
        for yi, xi in zip(y, x):
            yi += c * xi
        return None if z is None else self.dot(z, y)

    def negate(self, s):
        for t in s:
            t *= -1

    def scaled(self, s, a):
        return [a * t for t in s]

    def add_scaled(self, x, s, a):
        return [xi + a * si for xi, si in zip(x, s)]

    def project(self, x, g):
        for xi, gi in zip(x, g):
            C = xi.conj().T @ gi
            gi -= xi @ ((C + C.conj().T) / 2)

    def retract(self, y):
        out = []
        for yi in y:
            w, V = np.linalg.eigh(yi.conj().T @ yi)
            out.append(yi @ (V @ np.diag(1 / np.sqrt(w)) @ V.conj().T))
        return out

    def precondprep(self, x):
        if self.use_tpa:
            self.mean_kin = [np.sum(k[:, None] * np.abs(xi) ** 2, axis=0) for k, xi in zip(self.kin, x)]

    def ldiv(self, q):
        out = []
        for ik, qi in enumerate(q):
            f = 1.0 / self.kweights[ik]
            if self.use_tpa:
                mk = self.mean_kin[ik]
                out.append(f * (mk[None, :] / (mk[None, :] + self.kin[ik][:, None])) * qi)
            else:
                out.append(f * qi)
        return out


@pytest.mark.parametrize("prec_type", ["TPA", None])
def test_product_iteration_matches_the_oracle(prec_type):
    """The product's host-side iteration (lbfgs_iteration, over host versions of the device operations) against the
    independent oracle minimiser: the same energies over more iterations than the history length."""
    import dm_oracle
    from oracle.terms import Terms, energy_hamiltonian
    from oracle.scf import compute_density, random_orbitals
    b = _oracle_si()
    terms = Terms(b)
    f = b.model.filled_occupation
    rng = np.random.default_rng(5)
    psi0 = [random_orbitals(k.n_G, 4, rng) for k in b.kpoints]
    occ = [np.full(4, float(f)) for _ in b.kpoints]
    ops = NumpyOps(terms.kin, b.kweights, prec_type is not None)
    last = {}

    def value(psi):
        rho = compute_density(b, psi, occ)
        E, blocks = energy_hamiltonian(b, terms, psi, occ, rho)
        last.update(psi=psi, E=E, blocks=blocks)
        return E["total"]

    def value_gradient(psi):
        if last.get("psi") is not psi:
            value(psi)
        G = [2 * f * b.kweights[ik] * (blk @ p) for ik, (blk, p) in enumerate(zip(last["blocks"], psi))]
        ops.project(psi, G)
        ops.last_value = last["E"]["total"]
        return last["E"]["total"], G

    n = 14
    x = ops.retract([p.copy() for p in psi0])
    _, g = value_gradient(x)
    hist, energies = LBFGSHistory(), []
    for _ in range(n):
        x, g, E, _ = lbfgs_iteration(ops, hist, x, g, value, value_gradient)
        energies.append(E)
    ores = dm_oracle.direct_minimization(b, psi0, maxiter=n + 1, prec_type=prec_type, is_converged=lambda info: False)
    np.testing.assert_allclose(energies, ores["history_Etot"][:n], rtol=1e-12, atol=0)


def test_oracle_dm_matches_scf_spinless():
    # reference: test/scf_compare.jl "Compare different SCF algorithms (no spin, no temperature)"
    import dm_oracle
    from oracle import scf
    from oracle.scf import random_orbitals
    tol = 1e-7
    b = _oracle_si()
    ref = scf.self_consistent_field(b, tol=tol / 10)
    rng = np.random.default_rng(1234)
    psi0 = [random_orbitals(k.n_G, 4, rng) for k in b.kpoints]
    res = dm_oracle.direct_minimization(b, psi0, tol=tol)
    assert res["converged"]
    assert np.max(np.abs(res["rho"] - ref["rho"])) < 10 * tol
    assert abs(res["energies"]["total"] - ref["energies"]["total"]) < 1e-8


def test_oracle_dm_matches_scf_collinear():
    # reference: test/scf_compare.jl "collinear spin": DM started from the occupied orbitals of a one-step SCF
    import dm_oracle
    from oracle import scf
    from oracle.terms import guess_density
    tol = 1e-7
    b = _oracle_si(magnetic_moments=[1.0, 1.0])
    rho0 = guess_density(b, b.model.magnetic_moments)
    ref = scf.self_consistent_field(b, rho=rho0, tol=tol / 10)
    start = scf.self_consistent_field(b, rho=rho0, tol=tol, maxiter=1)
    sel = select_occupied_orbitals(b, [p.T for p in start["psi"]], start["occupation"])
    psi0 = [np.ascontiguousarray(p.T) for p in sel["psi"]]
    assert all(p.shape[1] == 4 for p in psi0)
    # the energy reaches rounding before Δρ < tol here: the minimiser ends on a failed line search, as Optim does
    res = dm_oracle.direct_minimization(b, psi0, tol=tol)
    assert np.max(np.abs(res["rho"] - ref["rho"])) < 10 * tol
    assert abs(res["energies"]["total"] - ref["energies"]["total"]) < 1e-8


def _dm_gloo_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import dftk_b200 as dftk
    comm = dftk.KpointComm.from_torch_distributed(with_nccl_id=False)
    basis = _StubBasis()
    Si = dftk.ElementPsp("Si")
    basis.model = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA())
    basis.comm_kpts = comm
    try:
        dftk.direct_minimization(basis)
        q.put((rank, comm.nranks, "no error"))
    except NotImplementedError as e:
        q.put((rank, comm.nranks, str(e)))
    dist.destroy_process_group()


def test_two_rank_kpoint_comm_is_refused_gloo():
    """A (k, spin)-sharded basis over two gloo ranks: every rank refuses, as the reference does under MPI."""
    import os
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_dm_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    assert out == [(0, 2, "Direct minimization with MPI is not supported yet"),
                   (1, 2, "Direct minimization with MPI is not supported yet")]
