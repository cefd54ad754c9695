"""NumPy direct minimisation on the oracle basis and terms (TEST INFRASTRUCTURE ONLY), written from the specification of
src/scf/direct_minimization.jl as the reference runs it (Optim.LBFGS(m=10) with the DMPreconditioner, the Stiefel manifold,
LineSearches.BackTracking(order=3) and InitialStatic) and independent of the product: nothing here is imported from
dftk_b200.  The energy and Hamiltonian are oracle.terms', the preconditioner is oracle.lobpcg.PreconditionerTPA divided by
the k-point weight, the retraction is Optim's Stiefel_SVD (U Vᴴ of the SVD), and ρout of the callback orthonormalises by QR
as the reference does.  Orbitals are (n_G, n_bands) column blocks, as everywhere in the oracle."""
import math
import numpy as np

from oracle.terms import Terms, energy_hamiltonian
from oracle.scf import compute_density
from oracle.lobpcg import PreconditionerTPA

M = 10


class LineSearchError(Exception):
    def __init__(self, alpha):
        super().__init__("BackTracking: no sufficient decrease within 1000 iterations")
        self.alpha = alpha


def _nanmin(a, b):
    return b if np.isnan(a) else (a if np.isnan(b) else min(a, b))


def _nanmax(a, b):
    return b if np.isnan(a) else (a if np.isnan(b) else max(a, b))


def backtracking(phi, phi0, dphi0, alpha=1.0, c1=1e-4, rho_hi=0.5, rho_lo=0.1, iterations=1000):
    """LineSearches.jl BackTracking, order 3, with Julia's IEEE semantics (x/0 is ±Inf or NaN, never an exception)."""
    with np.errstate(all="ignore"):
        f64 = np.float64
        phi0, dphi0 = f64(phi0), f64(dphi0)
        a_prev = a_cur = f64(alpha)
        phi_prev, phi_cur = phi0, f64(phi(a_cur))
        for _ in range(int(-np.log2(np.finfo(float).eps))):
            if np.isfinite(phi_cur):
                break
            a_prev, a_cur = a_cur, a_cur / 2
            phi_cur = f64(phi(a_cur))
        it = 0
        while phi_cur > phi0 + c1 * a_cur * dphi0:
            it += 1
            if it > iterations:
                raise LineSearchError(float(a_cur))
            if it == 1:
                a_new = -(dphi0 * a_cur * a_cur) / (2 * (phi_cur - phi0 - dphi0 * a_cur))
            else:
                r1 = phi_cur - phi0 - dphi0 * a_cur
                r0 = phi_prev - phi0 - dphi0 * a_prev
                den = f64(1) / (a_prev ** 2 * a_cur ** 2 * (a_cur - a_prev))
                ca = (a_prev ** 2 * r1 - a_cur ** 2 * r0) * den
                cb = (-a_prev ** 3 * r1 + a_cur ** 3 * r0) * den
                if abs(ca) <= np.finfo(float).eps:
                    a_new = dphi0 / (2 * cb)
                else:
                    a_new = (-cb + np.sqrt(max(cb * cb - 3 * ca * dphi0, f64(0)))) / (3 * ca)
            a_prev = a_cur
            a_cur = _nanmax(_nanmin(a_new, a_cur * rho_hi), a_cur * rho_lo)
            phi_prev, phi_cur = phi_cur, f64(phi(a_cur))
        return float(a_cur)


def direct_minimization(basis, psi0, tol=1e-6, maxiter=1000, prec_type="TPA", is_converged=None):
    """Returns psi, rho, energies, occupation, converged, n_iter, history_Etot, history_drho."""
    model = basis.model
    terms = Terms(basis)
    f = float(model.filled_occupation)
    nk = len(basis.kpoints)
    w = list(basis.kweights)
    n_bands = psi0[0].shape[1]
    occ = [np.full(n_bands, f) for _ in range(nk)]
    precs = [PreconditionerTPA(terms.kin[ik]) for ik in range(nk)] if prec_type is not None else None
    is_converged = is_converged or (lambda info: info["history_drho"][-1] < tol)

    def dot(a, b):
        return float(sum(np.real(np.vdot(x, y)) for x, y in zip(a, b)))

    def lin(a, ca, b, cb):
        return [ca * x + cb * y for x, y in zip(a, b)]

    def project(X, G):                                   # Optim.project_tangent!(Stiefel(), G, X)
        out = []
        for x, g in zip(X, G):
            XG = x.conj().T @ g
            out.append(g - x @ ((XG + XG.conj().T) / 2))
        return out

    def retract(Y):                                      # Optim.retract!(Stiefel_SVD(), X)
        out = []
        for y in Y:
            U, _, Vh = np.linalg.svd(y, full_matrices=False)
            out.append(U @ Vh)
        return out

    def precondprep(X):
        if precs is not None:
            for p, x in zip(precs, X):
                p.prep(x)

    def ldiv(Q):                                         # DMPreconditioner: P \ q / w_k
        if precs is None:
            return [q / w[ik] for ik, q in enumerate(Q)]
        return [precs[ik].ldiv(q) / w[ik] for ik, q in enumerate(Q)]

    def energy(X):
        rho = compute_density(basis, X, occ)
        E, blocks = energy_hamiltonian(basis, terms, X, occ, rho)
        return E, rho, blocks

    def projected_gradient(X, blocks):
        return project(X, [2 * f * w[ik] * (blocks[ik] @ x) for ik, x in enumerate(X)])

    # initial_state: retract, value and gradient (the gradient is projected by the manifold objective)
    x = retract([np.asarray(p, dtype=complex) for p in psi0])
    E, rho, blocks = energy(x)
    g = projected_gradient(x, blocks)
    hist_dx, hist_dg, hist_rho = [None] * M, [None] * M, [0.0] * M
    pseudo = 0
    history_Etot, history_drho = [], []
    converged = False
    n_iter = 0
    for _ in range(maxiter):
        n_iter += 1
        # update_state!(d, state, ::LBFGS)
        pseudo += 1
        g = project(x, g)
        precondprep(x)
        q = [t.copy() for t in g]
        alpha = {}
        for i in range(pseudo - 1, pseudo - M - 1, -1):
            if i < 1:
                continue
            j = (i - 1) % M
            alpha[i] = hist_rho[j] * dot(hist_dx[j], q)
            q = lin(q, 1.0, hist_dg[j], -alpha[i])
        s = ldiv(q)
        for i in range(pseudo - M, pseudo):
            if i < 1:
                continue
            j = (i - 1) % M
            beta = hist_rho[j] * dot(hist_dg[j], s)
            s = lin(s, 1.0, hist_dx[j], alpha[i] - beta)
        s = project(x, [-t for t in s])
        g_prev = g
        dphi0 = dot(g, s)
        if dphi0 >= 0:                                   # reset_search_direction!
            pseudo = 1
            s = [-t for t in ldiv(g)]
            dphi0 = dot(g, s)
        try:
            a = backtracking(lambda t: energy(retract(lin(x, 1.0, s, t)))[0]["total"], E["total"], dphi0)
        except LineSearchError as err:                   # Optim moves with the last step, then stops
            x = retract(lin(x, 1.0, s, err.alpha))
            break
        dx = [a * t for t in s]
        x = retract(lin(x, 1.0, dx, 1.0))
        # update_g!: value and projected gradient at the new point
        E, rho, blocks = energy(x)
        g = projected_gradient(x, blocks)
        # update_h!(d, state, ::LBFGS)
        dg = lin(g, 1.0, g_prev, -1.0)
        with np.errstate(divide="ignore"):
            r = np.float64(1.0) / np.float64(dot(dx, dg))
        if np.isinf(r):
            pseudo = 1
        else:
            j = (pseudo - 1) % M
            hist_dx[j], hist_dg[j], hist_rho[j] = dx, dg, float(r)
        # the reference's callback: stop one callback after convergence
        if converged:
            break
        rho_next = compute_density(basis, [np.linalg.qr(xk - sk)[0] for xk, sk in zip(x, s)], occ)
        history_drho.append(float(np.linalg.norm(rho_next - rho)) * math.sqrt(basis.dvol))
        history_Etot.append(E["total"])
        converged = bool(is_converged(dict(history_Etot=history_Etot, history_drho=history_drho, n_iter=n_iter)))
    rho = compute_density(basis, x, occ)
    E, _ = energy_hamiltonian(basis, terms, x, occ, rho)
    return dict(psi=x, rho=rho, energies=E, occupation=occ, converged=converged, n_iter=n_iter,
                history_Etot=history_Etot, history_drho=history_drho)
