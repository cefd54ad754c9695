"""direct_minimization: the ground state by direct minimisation of the Kohn–Sham energy over orthonormal orbitals
(host-side mirror of src/scf/direct_minimization.jl:68-201).

The reference hands the problem to Optim.jl with
`Optim.LBFGS(m=10, P=DMPreconditioner, precondprep=precondprep!, manifold=DMManifold, linesearch=BackTracking(),
alphaguess=InitialStatic())`; since a preconditioner is given, `scaleinvH0 = false`.  Optim sees one packed real vector,
so every inner product below is Re⟨a, b⟩ summed over all (k, spin) blocks.  The algorithm, restated:

Definitions
- Energy and gradient fg(ψ): ρ = compute_density(ψ, occ); E, ham = energy_hamiltonian(basis, ψ, occ, rho=ρ);
  G_k = 2 f w_k H_k ψ_k (f the filled occupation, w_k the k-point weight).
- Tangent projection (Optim.Stiefel): G ← G − X (XᴴG + GᴴX)/2 on each block.
- Retraction: the polar factor X (XᴴX)^{-1/2} (Optim's default Stiefel_SVD gives UVᴴ, the same matrix), from the
  eigendecomposition of the n_bands × n_bands Gram matrix.
- Preconditioner: precondprep!(P, x) sets each block's TPA mean_kin[n] = Σ_G kin_G |x_Gn|² (preconditioners.jl:75-77);
  ldiv!(s, P, q) is s_Gn = mean_kin[n]/(mean_kin[n] + kin_G) q_Gn / w_k (direct_minimization.jl:39-47).
  prec_type=None is the identity, still divided by w_k.
- The line search sees ϕ(α) = E(R(x + α s)); value_gradient(x) evaluates at R(x) and projects the gradient there.

One iteration (pseudo_iteration starts at 0):
1. pseudo_iteration += 1; project g at x; precondprep!(P, x).
2. Two-loop recursion over the indices pseudo_iteration−m … pseudo_iteration−1, skipping those < 1; the ring slot of an
   index is mod1(index, m).  Backward: α_i = ρ_i Re⟨dx_i, q⟩, q −= α_i dg_i.  Middle: s = P \\ q.
   Forward: β = ρ_i Re⟨dg_i, s⟩, s += (α_i − β) dx_i.  Finally s = −s, projected at x.
3. g_prev = g; dϕ0 = Re⟨g, s⟩.  If dϕ0 ≥ 0: pseudo_iteration = 1, s = −(P \\ g), dϕ0 = Re⟨g, s⟩.
4. BackTracking (order 3, c1 = 1e-4, ρ_hi = 0.5, ρ_lo = 0.1, at most 1000 iterations) from α = 1; see `backtracking`.
5. dx = α s; x = R(x + dx); g = the projected gradient at x.
6. dg = g − g_prev; ρ = 1/Re⟨dx, dg⟩.  If ρ is infinite: pseudo_iteration = 1 and nothing is stored; otherwise dx, dg
   and ρ go to ring slot mod1(pseudo_iteration, m).
7. Callback (direct_minimization.jl:122-146): ρout = density(ortho(ψ − s)) for the current point ψ and this iteration's
   direction s; ‖ρout − ρ‖ √dvol and E are appended to history_drho / history_Etot and `is_converged` is evaluated.
   As in the reference, the callback's info has rho = ρout and rho_in = ρ.
   Optim stops at the callback *after* the one that reports convergence, so one more iteration runs.

The accepted point of step 5 is the last point the line search evaluated, so its density and Hamiltonian are reused:
only the H apply of the gradient is added.

Memory: the history holds 2 m tall blocks (dx and dg), as in the reference; on the 128-atom silicon cell of bench.py that
is 20 × 0.55 GB.

Every tall-block operation is one libdftk_b200 call over all blocks of the rank (dm.cu); the reductions are deterministic,
so a run is reproducible bit for bit.
"""
import math
import time
import numpy as np
import torch

from .densities import compute_density
from .hamiltonian import energy_hamiltonian
from .scf import ScfConvergenceDensity
from . import device as _dev

M_HISTORY = 10


def _mod1(i, m):
    return (i - 1) % m + 1


def _nan_min(a, b):
    return b if math.isnan(a) else (a if math.isnan(b) else min(a, b))


def _nan_max(a, b):
    return b if math.isnan(a) else (a if math.isnan(b) else max(a, b))


class LineSearchFailed(RuntimeError):
    """LineSearches.LineSearchException: no sufficient decrease within the iteration limit; `alpha` is the last step."""

    def __init__(self, msg, alpha):
        super().__init__(msg)
        self.alpha = alpha


def backtracking(phi, phi_0, dphi_0, alpha_0=1.0, *, c_1=1e-4, rho_hi=0.5, rho_lo=0.1, iterations=1000):
    """LineSearches.BackTracking (order 3) as the reference's minimiser runs it.  Returns (α, ϕ(α)); raises
    LineSearchFailed after `iterations` shrinking steps.  The arithmetic is IEEE float64 as in Julia: a division by zero
    gives ±Inf or NaN, which the NaN-ignoring clipping then absorbs."""
    with np.errstate(all="ignore"):
        return _backtracking(phi, np.float64(phi_0), np.float64(dphi_0), np.float64(alpha_0), c_1, rho_hi, rho_lo, iterations)


def _backtracking(phi, phi_0, dphi_0, alpha_0, c_1, rho_hi, rho_lo, iterations):
    eps = np.finfo(float).eps
    iterfinitemax = -math.log2(eps)
    a1 = a2 = alpha_0
    phix_0, phix_1 = phi_0, np.float64(phi(a1))
    iterfinite = 0
    while not math.isfinite(phix_1) and iterfinite < iterfinitemax:
        iterfinite += 1
        a1 = a2
        a2 = a1 / 2
        phix_1 = np.float64(phi(a2))
    iteration = 0
    while phix_1 > phi_0 + c_1 * a2 * dphi_0:
        iteration += 1
        if iteration > iterations:
            raise LineSearchFailed(f"Linesearch failed to converge, reached maximum iterations {iterations}.", float(a2))
        if iteration == 1:
            a_tmp = -(dphi_0 * a2 ** 2) / (2 * (phix_1 - phi_0 - dphi_0 * a2))
        else:
            div = np.float64(1.0) / (a1 ** 2 * a2 ** 2 * (a2 - a1))
            a = (a1 ** 2 * (phix_1 - phi_0 - dphi_0 * a2) - a2 ** 2 * (phix_0 - phi_0 - dphi_0 * a1)) * div
            b = (-a1 ** 3 * (phix_1 - phi_0 - dphi_0 * a2) + a2 ** 3 * (phix_0 - phi_0 - dphi_0 * a1)) * div
            if abs(a) <= eps:
                a_tmp = dphi_0 / (2 * b)
            else:
                a_tmp = (-b + np.sqrt(max(b ** 2 - 3 * a * dphi_0, 0.0))) / (3 * a)
        a1 = a2
        a_tmp = _nan_min(a_tmp, a2 * rho_hi)
        a2 = _nan_max(a_tmp, a2 * rho_lo)
        phix_0, phix_1 = phix_1, np.float64(phi(a2))
    return float(a2), float(phix_1)


class LBFGSHistory:
    """The ring buffer of Optim's L-BFGS: slots 1..m, the slot of index i is mod1(i, m)."""

    def __init__(self, m=M_HISTORY):
        self.m = m
        self.pseudo_iteration = 0
        self.dx, self.dg, self.rho = [None] * (m + 1), [None] * (m + 1), [0.0] * (m + 1)

    def indices(self):
        """The history indices the two-loop recursion visits, oldest first."""
        p = self.pseudo_iteration
        return [i for i in range(p - self.m, p) if i >= 1]

    def store(self, dx, dg, dx_dot_dg):
        """Step 6.  Returns False (and resets) when ρ is infinite."""
        with np.errstate(divide="ignore"):
            rho = np.float64(1.0) / np.float64(dx_dot_dg)
        if math.isinf(rho):
            self.pseudo_iteration = 1
            return False
        s = _mod1(self.pseudo_iteration, self.m)
        self.dx[s], self.dg[s], self.rho[s] = dx, dg, float(rho)
        return True


def two_loop(ops, hist, g):
    """Step 2 without the final projection: s = −H g.  `ops` supplies the vector operations (module docstring)."""
    idx = hist.indices()
    q = ops.copy(g)
    alphas = {}
    if idx:
        # backward: each update is fused with the next dot product
        d = ops.dot(hist.dx[_mod1(idx[-1], hist.m)], q)
        for j in range(len(idx) - 1, -1, -1):
            sl = _mod1(idx[j], hist.m)
            alphas[idx[j]] = hist.rho[sl] * d
            nxt = hist.dx[_mod1(idx[j - 1], hist.m)] if j > 0 else None
            d = ops.axpy_dot(q, hist.dg[sl], -alphas[idx[j]], nxt)
    s = ops.ldiv(q)
    if idx:
        d = ops.dot(hist.dg[_mod1(idx[0], hist.m)], s)
        for j in range(len(idx)):
            sl = _mod1(idx[j], hist.m)
            beta = hist.rho[sl] * d
            nxt = hist.dg[_mod1(idx[j + 1], hist.m)] if j + 1 < len(idx) else None
            d = ops.axpy_dot(s, hist.dx[sl], alphas[idx[j]] - beta, nxt)
    ops.negate(s)
    return s


def lbfgs_iteration(ops, hist, x, g, value, value_gradient):
    """Steps 1-6 of one iteration.  `value(y)` is E at a retracted point y; `value_gradient(y)` returns (E, projected
    gradient) there.  Returns (x_new, g_new, E_new, s).  When the line search fails, Optim still moves to R(x + α s) with
    the last α tried and then stops: x_new is that point and g_new and E_new are None."""
    hist.pseudo_iteration += 1
    ops.project(x, g)
    ops.precondprep(x)
    s = two_loop(ops, hist, g)
    ops.project(x, s)
    g_prev = g
    phi_0 = ops.last_value
    dphi_0 = ops.dot(g, s)
    if dphi_0 >= 0:
        hist.pseudo_iteration = 1
        s = ops.ldiv(g)
        ops.negate(s)
        dphi_0 = ops.dot(g, s)

    last = {}

    def phi(a):
        last["alpha"], last["x"] = a, ops.retract(ops.add_scaled(x, s, a))
        return value(last["x"])

    try:
        alpha, _ = backtracking(phi, phi_0, dphi_0)
    except LineSearchFailed as e:
        return ops.retract(ops.add_scaled(x, s, e.alpha)), None, None, s
    dx = ops.scaled(s, alpha)
    # the line search ends on its last evaluation: R(x + α s) is that point, bit for bit
    x_new = last["x"] if last.get("alpha") == alpha else ops.retract(ops.add_scaled(x, s, alpha))
    E, g_new = value_gradient(x_new)
    dg = ops.copy(g_new)
    dxdg = ops.axpy_dot(dg, g_prev, -1.0, dx)
    hist.store(dx, dg, dxdg)
    return x_new, g_new, E, s


class DeviceOps:
    """The vector operations of the minimiser on lists of (n_bands, n_G) device tensors (one per k-block): each is one
    libdftk_b200 call over all blocks (dm.cu)."""

    def __init__(self, basis, n_bands, prec_type):
        self.kbs = basis.kblocks
        self.use_tpa = prec_type is not None
        self.inv_w = [1.0 / w for w in basis.kweights]
        self.mean_kin = torch.zeros((len(self.kbs), n_bands), dtype=torch.float64, device=basis.architecture.device)
        self.last_value = None

    def copy(self, a):
        return [t.clone() for t in a]

    def dot(self, a, b):
        return _dev.real_dots_multi(self.kbs, [(a, b)])[0]

    def axpy_dot(self, y, x, c, z=None):
        return _dev.axpy_dot_multi(self.kbs, y, x, c, z)

    def negate(self, s):
        _dev.axpy_dot_multi(self.kbs, s, s, -2.0)          # s + (−2) s = −s exactly

    def scaled(self, s, a):
        out = [torch.zeros_like(t) for t in s]
        _dev.axpy_dot_multi(self.kbs, out, s, a)
        return out

    def add_scaled(self, x, s, a):
        out = self.copy(x)
        _dev.axpy_dot_multi(self.kbs, out, s, a)
        return out

    def project(self, x, g):
        _dev.stiefel_project_multi(self.kbs, x, g)

    def retract(self, y):
        return _dev.stiefel_retract_multi(self.kbs, y)

    def precondprep(self, x):
        if self.use_tpa:
            _dev.tpa_multi(self.kbs, self.mean_kin, self.inv_w, True, X=x)

    def ldiv(self, q):
        s = [torch.empty_like(t) for t in q]
        _dev.tpa_multi(self.kbs, self.mean_kin, self.inv_w, self.use_tpa, Q=q, S=s)
        return s


def _occupation(basis, n_bands):
    f = basis.model.filled_occupation
    return [np.full(n_bands, float(f)) for _ in basis.kpoints]


class _Objective:
    """E(ψ) and its projected gradient; remembers the density and Hamiltonian of the last point it evaluated."""

    def __init__(self, basis, ops, occupation):
        self.basis, self.ops, self.occ = basis, ops, occupation
        self.last = None

    def _energy(self, psi):
        rho = compute_density(self.basis, psi, self.occ)
        energies, ham = energy_hamiltonian(self.basis, psi, self.occ, rho=rho)
        self.last = (psi, rho, energies, ham)
        return energies.total

    def value(self, psi):
        return self._energy(psi)

    def value_gradient(self, psi):
        if self.last is None or self.last[0] is not psi:
            self._energy(psi)
        _, _, energies, ham = self.last
        basis = self.basis
        f = basis.model.filled_occupation
        kbs = [ham[ik].bind() for ik in range(len(basis.kpoints))]
        G = [torch.empty_like(p) for p in psi]
        _dev.apply_h_multi(kbs, psi, G, scale=[2 * f * w for w in basis.kweights])
        self.ops.project(psi, G)
        self.ops.last_value = energies.total
        return energies.total, G


def energy_gradient(basis, psi, *, prec_type="TPA"):
    """E(ψ) and the Riemannian gradient (the tangent projection of 2 f w_k H_k ψ_k) at orthonormal orbitals ψ."""
    n_bands = psi[0].shape[0]
    ops = DeviceOps(basis, n_bands, prec_type)
    obj = _Objective(basis, ops, _occupation(basis, n_bands))
    return obj.value_gradient(psi)


def stiefel_retract(basis, psi):
    """The polar factor ψ (ψᴴψ)^{-1/2} of every block."""
    return _dev.stiefel_retract_multi(basis.kblocks, psi)


def select_occupied_orbitals(basis, psi, occupation, threshold=0.0):
    """orbitals.jl: keep the bands up to the last one whose occupation exceeds `threshold` on each k-point."""
    out_psi, out_occ = [], []
    for p, occ in zip(psi, occupation):
        occ = np.asarray(occ)
        above = np.nonzero(occ > threshold)[0]
        n = int(above[-1]) + 1 if len(above) else 0
        out_psi.append(p[:n].contiguous() if isinstance(p, torch.Tensor) else np.ascontiguousarray(p[:n]))
        out_occ.append(occ[:n].copy())
    return dict(psi=out_psi, occupation=out_occ)


def direct_minimization(basis, *, psi=None, tol=1e-6, is_converged=None, maxiter=1000, prec_type="TPA", callback=None,
                        seed=None):
    """direct_minimization.jl:68-201: minimise the Kohn–Sham energy over orthonormal orbitals (module docstring).
    Returns the keys of `self_consistent_field`'s result that apply, with `algorithm="DM"`."""
    model = basis.model
    if model.temperature != 0:
        raise ValueError("Direct minimization requires a model with zero temperature")
    if basis.comm_kpts.nranks > 1:
        raise NotImplementedError("Direct minimization with MPI is not supported yet")
    if getattr(basis, "comm_slab", None) is not None:
        raise NotImplementedError("Direct minimization does not support plane-wave slab distribution (comm_slab)")
    if basis.term("Hubbard") is not None:
        raise NotImplementedError("Direct minimization of a model with a Hubbard term is not supported")
    if prec_type not in ("TPA", None):
        raise ValueError(f"prec_type must be 'TPA' or None, not {prec_type!r}")
    start = time.time()
    n_bands = -(-model.n_electrons // (model.n_spin_components * model.filled_occupation))
    n_bands = int(n_bands)
    occupation = _occupation(basis, n_bands)
    if psi is None:
        from .eigen import _draw_seed
        gen = torch.Generator(device=basis.architecture.device)
        gen.manual_seed(int(seed if seed is not None else 0) + 7919 * basis.comm_kpts.rank)
        psi = _dev.random_orbitals_multi(basis.kblocks, n_bands, _draw_seed(gen))
    else:
        if len(psi) != len(basis.kpoints) or any(tuple(p.shape) != (n_bands, k.n_G) for p, k in zip(psi, basis.kpoints)):
            raise ValueError(f"psi must be a list of {len(basis.kpoints)} tensors of shape (n_bands={n_bands}, n_G)")
        psi = [torch.as_tensor(p, device=basis.architecture.device).to(torch.complex128).contiguous() for p in psi]
    is_converged = is_converged or ScfConvergenceDensity(tol)
    ops = DeviceOps(basis, n_bands, prec_type)
    obj = _Objective(basis, ops, occupation)
    hist = LBFGSHistory(M_HISTORY)

    x = ops.retract(psi)                       # value_gradient evaluates at R(x)
    _, g = obj.value_gradient(x)
    info = dict(basis=basis, history_Etot=[], history_drho=[], n_iter=0, converged=False, stage="iterate", algorithm="DM")
    converged = False
    for _ in range(maxiter):
        x, g, E, s = lbfgs_iteration(ops, hist, x, g, obj.value, obj.value_gradient)
        info["n_iter"] += 1
        if converged or g is None:          # stop at the callback after convergence, or on a failed line search
            break
        rho = obj.last[1]
        rho_out = compute_density(basis, ops.retract(ops.add_scaled(x, s, -1.0)), occupation)
        info["history_drho"].append(float((rho_out - rho).norm()) * math.sqrt(basis.dvol))
        info["history_Etot"].append(E)
        # the reference's keys (direct_minimization.jl:131): ρ is the density of the next step's orbitals, ρin the current one
        info.update(ham=obj.last[3], energies=obj.last[2], psi=x, occupation=occupation, rho=rho_out, rho_in=rho)
        converged = bool(is_converged(info))
        info["converged"] = converged
        if callback:
            callback(info)
    psi = x
    rho = compute_density(basis, psi, occupation)
    energies, ham = energy_hamiltonian(basis, psi, occupation, rho=rho)
    eigenvalues, psi = _rayleigh_ritz(basis, ham, psi)
    return dict(ham=ham, basis=basis, energies=energies, converged=converged, rho=rho, psi=psi, eigenvalues=eigenvalues,
                occupation=occupation, eF=None, n_iter=info["n_iter"], history_Etot=info["history_Etot"],
                history_drho=info["history_drho"], runtime_s=time.time() - start, stage="finalize", algorithm="DM")


def _rayleigh_ritz(basis, ham, psi):
    """The reference's final Rayleigh–Ritz: diagonalise ψᴴHψ per block, rotate ψ, return the eigenvalues."""
    kbs = [ham[ik].bind() for ik in range(len(basis.kpoints))]
    Hpsi = [torch.empty_like(p) for p in psi]
    _dev.apply_h_multi(kbs, psi, Hpsi)
    ctx = basis.architecture.ctx
    eigenvalues, out = [], []
    for p, hp in zip(psi, Hpsi):
        nb = p.shape[0]
        C = torch.zeros((nb, nb), dtype=torch.complex128, device=p.device)
        ctx.zgemm("C", p, hp, C)                                       # ψᴴ Hψ (column-major: C.T)
        w, V = np.linalg.eigh(C.T.cpu().numpy())
        eigenvalues.append(w)
        Vd = torch.as_tensor(np.ascontiguousarray(V.T), device=p.device)   # column-major V
        rot = torch.zeros_like(p)
        ctx.zgemm("N", p, Vd, rot)
        out.append(rot)
    return eigenvalues, out
