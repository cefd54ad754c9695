"""SCF driver restatement (oracle; test infrastructure only).

Follows src/scf/self_consistent_field.jl:80-289, scf_solvers.jl:76-102, anderson.jl,
mixing.jl:38-103, nbands_algorithm.jl, scf_callbacks.jl:191-230, densities.jl:13-57,
occupation.jl, symmetry.jl:282-357, eigen/diag.jl:9-65.
"""
import math
import numpy as np
from . import lobpcg as lob
from .terms import Terms, energy_hamiltonian, smearing_occupation
from .basis import index_G_vectors


# ------------------------------------------------------------------ orbitals.jl:82-87
def random_orbitals(n_G, howmany, rng):
    A = rng.standard_normal((n_G, howmany)) + 1j * rng.standard_normal((n_G, howmany))
    Q, _ = np.linalg.qr(A)
    return Q[:, :howmany]


# ------------------------------------------------------------------ diag.jl:9-65
def diagonalize_all_kblocks(blocks, nev, psiguess=None, tol=1e-6, miniter=1, maxiter=100,
                            n_conv_check=None, prec=True, rng=None, stats=None):
    rng = rng or np.random.default_rng(42)
    res = []
    for ik, blk in enumerate(blocks):
        n_G = blk.kpt.n_G
        if psiguess is not None:
            g = psiguess[ik]
            if g.shape[1] > nev:
                X0 = g[:, :nev]
            elif g.shape[1] == nev:
                X0 = g
            else:
                X0 = np.concatenate([g, rng.standard_normal((n_G, nev - g.shape[1]))
                                     + 1j * rng.standard_normal((n_G, nev - g.shape[1]))], axis=1)
                X0, _ = np.linalg.qr(X0)
        else:
            # interpolate_kpoint (interpolation.jl:96-115) only changes the start vector; the oracle
            # uses random orbitals for every k (converged results are guess-independent).
            X0 = random_orbitals(n_G, nev, rng)
        pre = lob.PreconditionerTPA(blk.kin) if prec and blk.kin is not None else None
        res.append(lob.lobpcg(blk, X0, pre, tol=tol, maxiter=maxiter, miniter=miniter,
                              n_conv_check=n_conv_check, rng=rng, stats=stats))
    return dict(λ=[r["λ"] for r in res], X=[r["X"] for r in res],
                residual_norms=[r["residual_norms"] for r in res],
                n_iter=[r["n_iter"] for r in res], converged=all(r["converged"] for r in res),
                n_matvec=sum(r["n_matvec"] for r in res))


# ------------------------------------------------------------------ occupation.jl
def _occupation_for(basis, eigenvalues, eF):
    m = basis.model
    invT = math.inf if m.temperature == 0 else 1 / m.temperature
    occ = []
    for ek in eigenvalues:
        with np.errstate(invalid="ignore"):
            x = (ek - eF) * invT
        x = np.where(np.isnan(x), 0.0, x)
        occ.append(m.filled_occupation * smearing_occupation(m.smearing if m.temperature > 0 else "None", x))
    return occ


def _excess(basis, eigenvalues, eF):
    occ = _occupation_for(basis, eigenvalues, eF)
    return sum(w * o.sum() for w, o in zip(basis.kweights, occ)) - basis.model.n_electrons


def compute_occupation(basis, eigenvalues, tol_n_elec=1e-6):
    m = basis.model
    n_fill = -(-m.n_electrons // (m.n_spin_components * m.filled_occupation))
    HOMO = max(ek[n_fill - 1] for ek in eigenvalues)
    lum = [ek[n_fill:].min() for ek in eigenvalues if len(ek) > n_fill]
    eF = (HOMO + min(lum)) / 2 if lum else HOMO + 1
    if m.temperature == 0:
        if abs(_excess(basis, eigenvalues, eF)) > tol_n_elec:
            raise RuntimeError("Unable to find non-fractional occupations; add a temperature")
    else:
        ex = _excess(basis, eigenvalues, eF)
        if abs(ex) >= tol_n_elec / 10:
            if ex < 0:
                lo, hi = eF, max(ek.max() for ek in eigenvalues) + 1
            else:
                lo, hi = min(ek.min() for ek in eigenvalues) - 1, eF
            for _ in range(200):                       # Roots.Bisection to atol=eps
                mid = (lo + hi) / 2
                if mid == lo or mid == hi:
                    break
                if _excess(basis, eigenvalues, mid) < 0:
                    lo = mid
                else:
                    hi = mid
            eF = (lo + hi) / 2
    return _occupation_for(basis, eigenvalues, eF), eF


# ------------------------------------------------------------------ symmetry.jl:282-357
def symmetrize_rho(basis, rho):
    syms = basis.symmetries
    if all(s.isone() for s in syms):
        return rho
    out = np.zeros_like(rho)
    for sp in range(rho.shape[0]):
        rf = basis.fft_cube(rho[sp])
        acc = np.zeros(basis.N, dtype=complex)
        for s in syms:
            invS = np.rint(np.linalg.inv(s.S)).astype(np.int64)
            idx = index_G_vectors(basis.fft_size, basis.G_all @ invS.T)
            val = np.where(idx >= 0, rf[np.maximum(idx, 0)], 0)
            if np.any(s.tau != 0):
                val = val * np.exp(-2j * math.pi * (basis.G_all @ s.tau))
            acc += val
        out[sp] = basis.irfft_cube(acc / len(syms))
    return out


# ------------------------------------------------------------------ densities.jl:13-57
def compute_density(basis, psi, occupation, occupation_threshold=0.0):
    rho = np.zeros((basis.model.n_spin_components, basis.N))
    for ik, kpt in enumerate(basis.kpoints):
        for n in range(psi[ik].shape[1]):
            if abs(occupation[ik][n]) < occupation_threshold:
                continue
            pr = basis.ifft_kpt(kpt, psi[ik][:, n], normalize=False)
            rho[kpt.spin] += (occupation[ik][n] * basis.kweights[ik] * basis.ifft_normalization ** 2
                              * np.abs(pr) ** 2)
    return symmetrize_rho(basis, rho)


# ------------------------------------------------------------------ nbands_algorithm.jl
class AdaptiveBands:
    def __init__(self, model, n_bands_converge=None, occupation_threshold=1e-6, gap_min=1e-2):
        def default_n_bands(factor):
            mn = -(-model.n_electrons // (model.n_spin_components * model.filled_occupation))
            f = 1.0 if model.temperature == 0 else factor
            return int(math.ceil(mn * f))
        self.n_bands_converge = n_bands_converge if n_bands_converge is not None else default_n_bands(1.05)
        self.n_bands_compute = max(3 + self.n_bands_converge, default_n_bands(1.20))
        self.occupation_threshold = occupation_threshold
        self.gap_min = gap_min

    def determine(self, occupation, eigenvalues, psi):
        if occupation is None:
            ncomp = self.n_bands_compute if psi is None else max(self.n_bands_compute, max(p.shape[1] for p in psi))
            return (self.n_bands_converge + self.n_bands_compute) // 2, ncomp
        def findlast(pred, arr):
            idx = [i for i, a in enumerate(arr) if pred(a)]
            return idx[-1] + 1 if idx else len(arr) + 1
        n_occ = max(findlast(lambda f: abs(f) >= self.occupation_threshold, o) for o in occupation)
        nconv = max(self.n_bands_converge, n_occ)
        ncomp_e = 0
        if eigenvalues is not None:
            vals = []
            for ek in eigenvalues:
                if nconv > len(ek):
                    vals.append(len(ek) + 1)
                else:
                    vals.append(findlast(lambda e: e <= ek[nconv - 1] + self.gap_min, ek))
            ncomp_e = max(vals)
        ncomp = max(self.n_bands_compute, ncomp_e, nconv + 3)
        if psi is not None:
            ncomp = max(ncomp, max(p.shape[1] for p in psi))
        return nconv, ncomp


# ------------------------------------------------------------------ anderson.jl
class Anderson:
    def __init__(self, m=10, maxcond=1e6, errorfactor=1e5):
        self.m, self.maxcond, self.errorfactor = m, maxcond, errorfactor
        self.xs, self.rs, self.errs = [], [], []

    def _push(self, x, r):
        self.xs.append(x.copy()); self.rs.append(r.copy()); self.errs.append(np.linalg.norm(r))
        if len(self.xs) > self.m:
            self.xs.pop(0); self.rs.pop(0); self.errs.pop(0)

    def __call__(self, x, alpha, Pf):
        shape = x.shape
        x, Pf = x.reshape(-1), Pf.reshape(-1)
        if not self.xs:
            self._push(x, Pf)
            return (x + alpha * Pf).reshape(shape)
        min_err = min(min(self.errs), np.linalg.norm(Pf))
        keep = [i for i in range(len(self.errs))
                if i == len(self.errs) - 1 or not self.errs[i] > self.errorfactor * min_err]
        self.xs = [self.xs[i] for i in keep]; self.rs = [self.rs[i] for i in keep]
        self.errs = [self.errs[i] for i in keep]
        Mm = np.stack(self.rs, axis=1) - Pf[:, None]
        while True:
            Q, Rr = np.linalg.qr(Mm)
            if Mm.shape[1] > 1 and np.linalg.cond(Rr) > self.maxcond:
                idrop = int(np.argmax(self.errs[:-1]))
                for lst in (self.xs, self.rs, self.errs):
                    lst.pop(idrop)
                Mm = np.delete(Mm, idrop, axis=1)
                continue
            break
        xn = x + alpha * Pf
        betas = -np.linalg.lstsq(Mm, Pf, rcond=None)[0]
        for ib, b in enumerate(betas):
            xn = xn + b * (self.xs[ib] - x + alpha * (self.rs[ib] - Pf))
        self._push(x, Pf)
        return xn.reshape(shape)


def kerker_mix(basis, dF, kTF=0.8):
    """mixing.jl:61-103 (ΔDOS_Ω = 0)."""
    G2 = np.sum(basis.G_cart ** 2, axis=1)
    tot = dF.sum(axis=0)
    tf = basis.fft_cube(tot) * G2 / (kTF ** 2 + G2)
    dtot = basis.irfft_cube(basis.enforce_real(tf))
    dtot += tot.mean() - dtot.mean()
    if dF.shape[0] == 1:
        return dtot[None, :]
    spin = dF[0] - dF[1]
    return np.stack([(dtot + spin) / 2, (dtot - spin) / 2])


# ------------------------------------------------------------------ LdosMixing: mixing.jl:205-292, chi0models.jl:20-41, dos.jl:43-65
def gmres(apply, b, rtol=0.01, atol=1e-12, krylovdim=30, maxiter=100):
    """Restarted GMRES from x0 = 0 (modified Gram-Schmidt Arnoldi, Givens rotations), the published algorithm behind the
    `KrylovKit.linsolve(f, b; rtol, ishermitian=false)` call of mixing.jl:283 (KrylovKit is a third-party dependency, compat
    "0.8.3, 0.9, 0.10", not under the DFTK.jl tree): stop when the residual estimate is below max(atol, rtol ||b||)."""
    b = np.asarray(b, dtype=float)
    shape = b.shape
    b = b.reshape(-1)
    x = np.zeros_like(b)
    tol = max(atol, rtol * np.linalg.norm(b))
    r = b.copy()
    beta = np.linalg.norm(r)
    n_apply = 0
    for _restart in range(maxiter):
        if beta <= tol:
            break
        V = [r / beta]
        H = np.zeros((krylovdim + 1, krylovdim))
        cs, sn = np.zeros(krylovdim), np.zeros(krylovdim)
        g = np.zeros(krylovdim + 1)
        g[0] = beta
        k_used = 0
        for k in range(krylovdim):
            w = apply(V[k].reshape(shape)).reshape(-1)
            n_apply += 1
            for j in range(k + 1):
                H[j, k] = np.dot(V[j], w)
                w = w - H[j, k] * V[j]
            H[k + 1, k] = np.linalg.norm(w)
            for j in range(k):
                t = cs[j] * H[j, k] + sn[j] * H[j + 1, k]
                H[j + 1, k] = -sn[j] * H[j, k] + cs[j] * H[j + 1, k]
                H[j, k] = t
            den = math.hypot(H[k, k], H[k + 1, k])
            cs[k], sn[k] = H[k, k] / den, H[k + 1, k] / den
            H[k, k] = den
            H[k + 1, k] = 0.0
            g[k + 1] = -sn[k] * g[k]
            g[k] = cs[k] * g[k]
            k_used = k + 1
            if abs(g[k + 1]) <= tol:
                break
            V.append(w / np.linalg.norm(w))
        y = np.linalg.solve(np.triu(H[:k_used, :k_used]), g[:k_used])
        for j in range(k_used):
            x = x + y[j] * V[j]
        r = b - apply(x.reshape(shape)).reshape(-1)
        n_apply += 1
        beta = np.linalg.norm(r)
    return x.reshape(shape), dict(converged=beta <= tol, n_apply=n_apply, residual=beta)


def compute_ldos(basis, eF, eigenvalues, psi, temperature, weight_threshold=np.finfo(float).eps):
    """dos.jl:43-65 with Gaussian smearing: occupation_derivative f'(x) = -exp(-x²)/sqrt(pi)."""
    filled = basis.model.filled_occupation
    w = [-filled / temperature * (-np.exp(-((np.asarray(e) - eF) / temperature) ** 2) / math.sqrt(math.pi)) for e in eigenvalues]
    return compute_density(basis, psi, w, weight_threshold)


def ldos_mix(basis, dF, terms, info, rtol=0.01):
    """mix_density(::χ0Mixing with [LdosModel()], RPA = true), mixing.jl:262-292."""
    m = basis.model
    Tm = max(m.temperature, min(0.1, 100 * m.temperature))         # default_smearing_temperature, mixing.jl:296-301
    if Tm == 0:
        return dF
    ldos = compute_ldos(basis, info["eF"], info["eigenvalues"], info["psi"], Tm)
    if np.abs(ldos).max() < math.sqrt(np.finfo(float).eps):
        return dF
    tdos = ldos.sum() * basis.dvol
    green = terms.green

    def adjoint(d):
        dV = np.zeros_like(d)
        if green is not None:
            dV[:] = basis.irfft_cube(green * basis.fft_cube(d.sum(axis=0)))[None, :]      # Hartree kernel on the total density
        dV = dV - dV.mean()
        deF = np.sum(ldos * dV) * basis.dvol
        e = d - (-ldos * dV + ldos * deF / tdos)                                          # εδF .-= χ0 δV
        return e - e.mean()

    dc = dF.mean()
    x, st = gmres(adjoint, dF - dc, rtol=rtol)
    return x + dc


# ------------------------------------------------------------------ self_consistent_field.jl
def self_consistent_field(basis, rho=None, tol=1e-6, maxiter=100, damping=0.8, mixing="simple",
                          nbandsalg=None, is_converged=None, rng=None, callback=None,
                          diagtol_first=None, stats=None, anderson_m=10):
    from .terms import guess_density
    model = basis.model
    terms = Terms(basis)
    rng = rng or np.random.default_rng(7)
    nbandsalg = nbandsalg or AdaptiveBands(model)
    rho = guess_density(basis) if rho is None else rho
    info = dict(psi=None, occupation=None, eigenvalues=None, eF=None, n_iter=0, n_matvec=0,
                history_Etot=[], history_drho=[], converged=False)
    acc = Anderson(m=anderson_m)
    diagtol_max = 0.005
    if is_converged is None:
        is_converged = lambda inf: inf["history_drho"][-1] < tol

    if diagtol_first is None and not any(t in model.terms for t in ("Hartree", "Xc")):
        diagtol_first = tol / 5          # default_diagtolalg, scf_callbacks.jl:220-229 (no nonlinear term)

    def fixpoint_map(rho_in):
        # determine_diagtol, scf_callbacks.jl:198-212, is handed the info of the PREVIOUS step
        # (self_consistent_field.jl:198-203): n_iter is 0 and 1 for the first two steps
        if info["n_iter"] <= 1:
            dt = min(6 * diagtol_max if diagtol_first is None else diagtol_first, 5 * diagtol_max)
        else:
            dt = min(max(min(info["history_drho"]) * 0.2, 100 * np.finfo(float).eps), diagtol_max)
        info["n_iter"] += 1
        _E, blocks = energy_hamiltonian(basis, terms, info["psi"], info["occupation"], rho_in,
                                        info["eigenvalues"], info["eF"])
        nconv, ncomp = nbandsalg.determine(info["occupation"], info["eigenvalues"], info["psi"])
        if info["psi"] is not None:
            ncomp = max(ncomp, max(p.shape[1] for p in info["psi"]))
        eig = diagonalize_all_kblocks(blocks, ncomp, psiguess=info["psi"], tol=dt, miniter=1,
                                      n_conv_check=nconv, rng=rng, stats=stats)
        occ, eF = compute_occupation(basis, eig["λ"], tol_n_elec=nbandsalg.occupation_threshold)
        rho_out = compute_density(basis, eig["X"], occ, nbandsalg.occupation_threshold)
        info.update(psi=eig["X"], eigenvalues=eig["λ"], occupation=occ, eF=eF, rho_out=rho_out,
                    n_matvec=info["n_matvec"] + eig["n_matvec"], diag=eig, diagtol=dt,
                    n_bands_converge=nconv)
        E, _ = energy_hamiltonian(basis, terms, eig["X"], occ, rho_out, eig["λ"], eF, only_energy=True)
        drho = rho_out - rho_in
        info["energies"] = E
        info["history_Etot"].append(E["total"])
        info["history_drho"].append(float(np.linalg.norm(drho) * math.sqrt(basis.dvol)))
        if mixing == "simple":
            mixed = drho
        elif mixing == "kerker":
            mixed = kerker_mix(basis, drho)
        elif mixing == "ldos":             # the reference default (self_consistent_field.jl:177)
            mixed = ldos_mix(basis, drho, terms, info)
        else:
            raise ValueError(mixing)
        info["converged"] = bool(is_converged(info))
        if callback:
            callback(info)
        return rho_in + mixed

    x = rho
    for _i in range(maxiter):
        fx = fixpoint_map(x)
        if info["converged"]:
            break
        x = acc(x, damping, fx - x)
    rho_f = info["rho_out"]
    E, blocks = energy_hamiltonian(basis, terms, info["psi"], info["occupation"], rho_f,
                                   info["eigenvalues"], info["eF"])
    return dict(energies=E, ham=blocks, rho=rho_f, psi=info["psi"], eigenvalues=info["eigenvalues"],
                occupation=info["occupation"], eF=info["eF"], converged=info["converged"],
                n_iter=info["n_iter"], n_matvec=info["n_matvec"], history_Etot=info["history_Etot"],
                history_drho=info["history_drho"], terms=terms, basis=basis)
