"""self_consistent_field and friends (host-side mirror of src/scf/self_consistent_field.jl:80-289,
scf_solvers.jl:76-102, anderson.jl, mixing.jl:38-103, nbands_algorithm.jl, scf_callbacks.jl:191-230).

Host orchestration only: the density, potentials, orbitals and Anderson history stay on the device;
every orbital-sized operation is a libdftk_b200 call."""
import math
import time
import numpy as np
import torch

from .hamiltonian import energy_hamiltonian, energy, ksum_energy_partials
from .eigen import lobpcg_hyper, diagonalize_all_kblocks
from .occupation import compute_occupation, gather_eigenvalues
from .densities import compute_density
from .terms import guess_density


class AdaptiveBands:
    """nbands_algorithm.jl:57-109."""

    def __init__(self, model, *, n_bands_converge=None, occupation_threshold=1e-6, gap_min=1e-2,
                 temperature_factor_converge=1.05, temperature_factor_compute=1.20):
        def default_n_bands(factor):
            mn = -(-model.n_electrons // (model.n_spin_components * model.filled_occupation))
            return int(math.ceil(mn * (1.0 if model.temperature == 0 else factor)))
        self.n_bands_converge = default_n_bands(temperature_factor_converge) if n_bands_converge is None else n_bands_converge
        self.n_bands_compute = max(3 + self.n_bands_converge, default_n_bands(temperature_factor_compute))
        self.occupation_threshold, self.gap_min = occupation_threshold, gap_min

    def determine_n_bands(self, occupation, eigenvalues, psi):
        if occupation is None:
            ncomp = self.n_bands_compute if psi is None else max(self.n_bands_compute, max(p.shape[0] for p in psi))
            return (self.n_bands_converge + self.n_bands_compute) // 2, ncomp

        def findlast(pred, arr):
            idx = [i for i, a in enumerate(arr) if pred(a)]
            return idx[-1] + 1 if idx else len(arr) + 1
        n_occ = max(findlast(lambda f: abs(f) >= self.occupation_threshold, o) for o in occupation)
        nconv = max(self.n_bands_converge, n_occ)
        ncomp_e = 0
        if eigenvalues is not None:
            ncomp_e = max(len(ek) + 1 if nconv > len(ek) else
                          findlast(lambda e, ek=ek: e <= ek[nconv - 1] + self.gap_min, ek) for ek in eigenvalues)
        ncomp = max(self.n_bands_compute, ncomp_e, nconv + 3)
        if psi is not None:
            ncomp = max(ncomp, max(p.shape[0] for p in psi))
        return nconv, ncomp


class FixedBands:
    def __init__(self, n_bands_converge, n_bands_compute=None, occupation_threshold=1e-6):
        self.n_bands_converge = n_bands_converge
        self.n_bands_compute = n_bands_compute if n_bands_compute is not None else n_bands_converge + 3
        self.occupation_threshold = occupation_threshold

    def determine_n_bands(self, occupation, eigenvalues, psi):
        return self.n_bands_converge, self.n_bands_compute


class AdaptiveDiagtol:
    """scf_callbacks.jl:191-212."""

    def __init__(self, ratio_rhodiff=0.2, diagtol_min=None, diagtol_max=0.005, diagtol_first=None):
        self.ratio, self.dmin, self.dmax = ratio_rhodiff, diagtol_min, diagtol_max
        self.dfirst = 6 * diagtol_max if diagtol_first is None else diagtol_first

    def determine_diagtol(self, info):
        if info["n_iter"] <= 1:
            return min(self.dfirst, 5 * self.dmax)
        d = min(info["history_drho"]) * self.ratio
        dmin = 100 * np.finfo(float).eps if self.dmin is None else self.dmin
        return min(max(d, dmin), self.dmax)


class ScfConvergenceDensity:
    def __init__(self, tol):
        self.tol = tol

    def __call__(self, info):
        return info["history_drho"][-1] < self.tol


class ScfConvergenceEnergy:
    def __init__(self, tol):
        self.tol = tol

    def __call__(self, info):
        h = info["history_Etot"]
        return len(h) > 1 and abs(h[-1] - h[-2]) < self.tol


class SimpleMixing:
    def mix_density(self, basis, dF, **kw):
        return dF


class KerkerMixing:
    """mixing.jl:61-103 (ΔDOS_Ω = 0)."""

    def __init__(self, kTF=0.8):
        self.kTF = kTF

    def mix_density(self, basis, dF, **kw):
        G2 = (basis.G_vectors_cart ** 2).sum(dim=1)
        tot = dF.sum(dim=0)
        tf = basis.fft(tot).reshape(-1) * G2 / (self.kTF ** 2 + G2)
        dtot = basis.irfft(basis.enforce_real(tf)).reshape(-1)
        dtot = dtot + (tot.mean() - dtot.mean())
        if dF.shape[0] == 1:
            return dtot[None, :]
        spin = dF[0] - dF[1]
        return torch.stack([(dtot + spin) / 2, (dtot - spin) / 2])


class LdosMixing:
    """LdosMixing = χ0Mixing([LdosModel()], RPA = true), the reference's default mixing (self_consistent_field.jl:177;
    mixing.jl:205-292, chi0models.jl:20-41): solve (1 - χ0 v_c)^† δρ = δF by GMRES with
    χ0(r, r') = -D_loc(r) δ(r, r') + D_loc(r) D_loc(r') / D, the local density of states from one more density pass with
    the weights -f'((ε - εF)/T_mix)/T_mix (compute_ldos, dos.jl:43-65; Gaussian smearing at T_mix = max(T, min(0.1, 100 T))).
    Degenerates to simple mixing at T = 0.  Everything stays on the device: the LDOS is a `compute_density` call (batched
    FFT pipeline + NCCL allreduce + symmetrisation), the Hartree kernel two cube FFTs, the Krylov dot products one fused
    Gram launch per Arnoldi step."""

    def __init__(self, rtol=0.01, krylovdim=30, maxiter=100, temperature=None):
        self.rtol, self.krylovdim, self.maxiter, self.temperature = rtol, krylovdim, maxiter, temperature
        self.last = None

    def mix_density(self, basis, dF, *, psi=None, eigenvalues=None, eF=None, **kw):
        m = basis.model
        Tm = self.temperature if self.temperature is not None else max(m.temperature, min(0.1, 100 * m.temperature))
        if Tm == 0 or psi is None or eigenvalues is None or eF is None:
            return dF
        ldos = compute_ldos(basis, eF, eigenvalues, psi, temperature=Tm)
        if float(ldos.abs().max()) < math.sqrt(np.finfo(float).eps):
            return dF
        tdos = float(ldos.sum()) * basis.dvol
        hartree = basis.term("Hartree")
        green = hartree.poisson_green_coeffs if hartree is not None else None
        shape = dF.shape

        def adjoint(d):          # ε^† δF = δF - χ0 (v_c δF), both DC components removed (mixing.jl:268-278)
            d = d.reshape(shape)
            if green is not None:
                dV = basis.irfft(green * basis.fft(d.sum(dim=0)).reshape(-1)).reshape(1, -1).expand(shape[0], -1)
            else:
                dV = torch.zeros_like(d)
            dV = dV - dV.mean()
            deF = float((ldos * dV).sum()) * basis.dvol
            e = d - (-ldos * dV + ldos * (deF / tdos))
            return (e - e.mean()).reshape(-1)

        dc = dF.mean()
        x, self.last = _gmres(basis.architecture.ctx, adjoint, (dF - dc).reshape(-1), self.rtol, 1e-12, self.krylovdim,
                              self.maxiter)
        if not self.last["converged"]:
            import warnings
            warnings.warn("LDOS mixing GMRES not converged")
        return x.reshape(shape) + dc


def compute_ldos(basis, eF, eigenvalues, psi, *, temperature, weight_threshold=np.finfo(float).eps):
    """dos.jl:43-65 with Gaussian smearing (occupation_derivative f'(x) = -exp(-x²)/sqrt(π)): a density pass with the
    weights -filled/T f'((ε - εF)/T); the k-sum, the allreduce and the symmetrisation come with compute_density."""
    filled = basis.model.filled_occupation
    w = [filled / temperature * np.exp(-((np.asarray(e) - eF) / temperature) ** 2) / math.sqrt(math.pi) for e in eigenvalues]
    w = [wk[:p.shape[0]] for wk, p in zip(w, psi)]
    return compute_density(basis, psi, w, occupation_threshold=weight_threshold)


def _gmres(ctx, apply, b, rtol, atol, krylovdim, maxiter):
    """Restarted GMRES from x0 = 0 (Arnoldi + Givens rotations), the algorithm behind the reference's
    `KrylovKit.linsolve(f, b; rtol, ishermitian=false)` (mixing.jl:283).  Vectors are flat float64 device tensors; the
    projections of an Arnoldi step onto all previous vectors are ONE fused Gram launch (dftk_b200_tall_gram)."""
    n = b.numel()
    npad = n + (n & 1)

    def pad(v):
        return v if npad == n else torch.cat([v, v.new_zeros(1)])

    tol = max(atol, rtol * float(b.norm()))
    x = torch.zeros_like(b)
    r = b.clone()
    beta = float(r.norm())
    n_apply = 0
    for _restart in range(maxiter):
        if beta <= tol:
            break
        V = torch.zeros((krylovdim + 1, npad), dtype=torch.float64, device=b.device)
        V[0, :n] = r / beta
        H = np.zeros((krylovdim + 1, krylovdim))
        cs, sn, g = np.zeros(krylovdim), np.zeros(krylovdim), np.zeros(krylovdim + 1)
        g[0] = beta
        k_used = 0
        for k in range(krylovdim):
            w = pad(apply(V[k, :n]))
            n_apply += 1
            for _pass in range(2):                                 # classical Gram-Schmidt, twice (as stable as MGS)
                h = ctx.real_gram(V[:k + 1], w[None, :].contiguous())[:, 0]
                w = w - torch.as_tensor(h, device=b.device) @ V[:k + 1]
                H[:k + 1, k] += h
            H[k + 1, k] = float(w.norm())
            for j in range(k):
                t = cs[j] * H[j, k] + sn[j] * H[j + 1, k]
                H[j + 1, k] = -sn[j] * H[j, k] + cs[j] * H[j + 1, k]
                H[j, k] = t
            den = math.hypot(H[k, k], H[k + 1, k])
            wnorm = H[k + 1, k]
            cs[k], sn[k] = H[k, k] / den, H[k + 1, k] / den
            H[k, k], H[k + 1, k] = den, 0.0
            g[k + 1] = -sn[k] * g[k]
            g[k] = cs[k] * g[k]
            k_used = k + 1
            if abs(g[k + 1]) <= tol or wnorm == 0.0:
                break
            V[k + 1] = w / wnorm
        y = np.linalg.solve(np.triu(H[:k_used, :k_used]), g[:k_used])
        x = x + (torch.as_tensor(y, device=b.device) @ V[:k_used])[:n]
        r = b - apply(x)
        n_apply += 1
        beta = float(r.norm())
    return x, dict(converged=beta <= tol, n_apply=n_apply, residual=beta)


class AndersonAcceleration:
    """anderson.jl:42-130, history kept on the device.  The least-squares problem min |Pf + M β| is solved from the Gram
    matrix of [M, Pf] -- one fused launch over the N_fft-sized history (dftk_b200_tall_gram) instead of a QR factorisation
    of the N_fft × m matrix -- with one step of iterative refinement on the true residual (a second launch), which
    restores the accuracy the normal equations lose when cond(M) approaches maxcond; cond(M) = sqrt(cond(M'M))."""

    def __init__(self, m=10, maxcond=1e6, errorfactor=1e5, ctx=None):
        self.m, self.maxcond, self.errorfactor, self.ctx = m, maxcond, errorfactor, ctx
        self.xs, self.rs, self.errs = [], [], []

    def _push(self, x, r):
        self.xs.append(x.clone()); self.rs.append(r.clone()); self.errs.append(float(r.norm()))
        if len(self.xs) > self.m:
            self.xs.pop(0); self.rs.pop(0); self.errs.pop(0)

    def _gram(self, A, B):
        if self.ctx is None or not A.is_cuda:
            return (A @ B.T).cpu().numpy()            # host tensors (CPU-only unit tests of the host logic)
        n = A.shape[1]
        if n & 1:
            A = torch.cat([A, A.new_zeros(A.shape[0], 1)], dim=1)
            B = torch.cat([B, B.new_zeros(B.shape[0], 1)], dim=1)
        return self.ctx.real_gram(A.contiguous(), B.contiguous())

    def __call__(self, x, alpha, Pf):
        shape = x.shape
        x, Pf = x.reshape(-1), Pf.reshape(-1)
        if self.m == 0 or self.errorfactor <= 1 or self.maxcond <= 1:
            return (x + alpha * Pf).reshape(shape)
        if not self.xs:
            self._push(x, Pf)
            return (x + alpha * Pf).reshape(shape)
        min_err = min(min(self.errs), float(Pf.norm()))
        keep = [i for i in range(len(self.errs)) if i == len(self.errs) - 1 or not self.errs[i] > self.errorfactor * min_err]
        self.xs, self.rs, self.errs = ([l[i] for i in keep] for l in (self.xs, self.rs, self.errs))
        M = torch.stack(self.rs, dim=0) - Pf[None, :]              # rows M_j = Pf_j - Pf
        Gext = self._gram(torch.cat([M, Pf[None, :]], dim=0), torch.cat([M, Pf[None, :]], dim=0))
        k = M.shape[0]
        G, g = Gext[:k, :k], Gext[:k, k]
        cols = list(range(k))

        def cond(idx):
            ev = np.linalg.eigvalsh(G[np.ix_(idx, idx)])
            return math.inf if ev[0] <= 0 else math.sqrt(ev[-1] / ev[0])

        while len(cols) > 1 and cond(cols) > self.maxcond:
            idrop = int(np.argmax(self.errs[:-1]))
            for l in (self.xs, self.rs, self.errs):
                l.pop(idrop)
            cols.pop(idrop)
        Mk = M[cols]
        Gk = G[np.ix_(cols, cols)]
        betas = -np.linalg.solve(Gk, g[cols])
        res = Pf + torch.as_tensor(betas, device=Pf.device) @ Mk      # refinement on the true least-squares residual
        betas = betas - np.linalg.solve(Gk, self._gram(Mk, res[None, :])[:, 0])
        xn = x + alpha * Pf
        for ib, b in enumerate(betas.tolist()):
            xn = xn + b * (self.xs[ib] - x + alpha * (self.rs[ib] - Pf))
        self._push(x, Pf)
        return xn.reshape(shape)


def next_density(ham, nbandsalg, *, eigensolver=lobpcg_hyper, psi=None, eigenvalues=None, occupation=None,
                 tol=1e-6, miniter=1, maxiter=100, generator=None, fermialg=None):
    """self_consistent_field.jl:80-129.  `eigenvalues` / `occupation` drive the band-count heuristics: pass the lists
    over ALL (k, spin) blocks (the `*_global` entries of the previous result) so that every rank takes the same
    decision without the mpi_max of self_consistent_field.jl:98.

    Collectives of the sharded path: one allgather (eigenvalues + solver statistics) and one allreduce (density with
    the k-summed band-energy partials packed behind it)."""
    basis = ham.basis
    nconv, ncomp = nbandsalg.determine_n_bands(occupation, eigenvalues, psi)
    if psi is not None:
        ncomp = max(ncomp, max(p.shape[0] for p in psi))
    eig = diagonalize_all_kblocks(eigensolver, ham, ncomp, psiguess=psi, n_conv_check=nconv, tol=tol,
                                  miniter=miniter, maxiter=maxiter, generator=generator)
    ev_g, w_g, stats = gather_eigenvalues(basis, eig["λ"], stats=[eig["n_matvec"], 1.0 if eig["converged"] else 0.0])
    eig["converged"] = bool(np.all(stats[:, 1] > 0.5))
    if not eig["converged"]:
        import warnings
        warnings.warn(f"Eigensolver not converged, n_iter={eig['n_iter']}")
    occ, eF, occ_g = compute_occupation(basis, eig["λ"], fermialg=fermialg, tol_n_elec=nbandsalg.occupation_threshold,
                                        gathered=(ev_g, w_g), return_global=True)
    names, partials = ksum_energy_partials(basis, eig["X"], occ, eig["λ"], eF)
    hub = basis.term("Hubbard")
    n_hub = None
    if hub is not None:
        # this rank's partial of the Hubbard occupation rides behind the density in the same allreduce
        n_hub = hub.local_occupation(basis, eig["X"], occ)
        partials = np.concatenate([partials, n_hub.real.ravel(), n_hub.imag.ravel()])
    rho, totals = compute_density(basis, eig["X"], occ, occupation_threshold=nbandsalg.occupation_threshold,
                                  packed_sums=partials)
    if n_hub is not None:
        tail = totals[len(names):]
        n_hub = (tail[:n_hub.size] + 1j * tail[n_hub.size:]).reshape(n_hub.shape)
        basis._hubbard_cache = dict(psi=eig["X"], occupation=occ, n=n_hub)
        totals = totals[:len(names)]
    basis._ksum_cache = dict(psi=eig["X"], occupation=occ, eF=eF, totals=dict(zip(names, totals)))
    return dict(psi=eig["X"], eigenvalues=eig["λ"], occupation=occ, eF=eF, rho=rho, diagonalization=eig,
                n_bands_converge=nconv, n_matvec=int(round(float(np.sum(stats[:, 0])))),
                eigenvalues_global=ev_g, occupation_global=occ_g)


def self_consistent_field(basis, *, rho=None, psi=None, tol=1e-6, is_converged=None, maxiter=100,
                          mixing=None, damping=0.8, eigensolver=lobpcg_hyper, diagtolalg=None, nbandsalg=None,
                          callback=None, compute_consistent_energies=True, seed=None, anderson_m=10, hubbard_n=None,
                          fermialg=None):
    """self_consistent_field.jl:19-45,168-289.  `hubbard_n`: the starting Hubbard occupation of a model with a Hubbard
    term (None: the first Hamiltonian has no Hubbard operator).  Each step's Hamiltonian uses the previous step's
    occupation; it is recomputed from the new orbitals after every density update, never mixed, and returned.
    `fermialg`: the Fermi-level search, FermiBisection() or FermiTwoStage() (default: default_fermialg(model.smearing))."""
    model = basis.model
    hub = basis.term("Hubbard")
    start = time.time()
    rho = guess_density(basis) if rho is None else rho
    mixing = mixing or LdosMixing()        # the reference default (self_consistent_field.jl:177); simple mixing at T = 0
    nbandsalg = nbandsalg or AdaptiveBands(model)
    if diagtolalg is None:       # default_diagtolalg, scf_callbacks.jl:220-229
        nonlinear = any(t in model.term_types for t in ("Hartree", "Xc"))
        diagtolalg = AdaptiveDiagtol() if nonlinear else AdaptiveDiagtol(diagtol_first=tol / 5)
    is_converged = is_converged or ScfConvergenceDensity(tol)
    gen = torch.Generator(device=basis.architecture.device)
    gen.manual_seed(int(seed if seed is not None else 0) + 7919 * basis.comm_kpts.rank)   # same `seed` on every rank
    info = dict(basis=basis, rho=rho, psi=psi, occupation=None, eigenvalues=None, eF=None, n_iter=0, n_matvec=0,
                eigenvalues_global=None, occupation_global=None, hubbard_n=hubbard_n,
                converged=False, history_Etot=[], history_drho=[], stage="iterate", algorithm="SCF")
    acc = AndersonAcceleration(m=anderson_m, ctx=basis.architecture.ctx)

    def fixpoint_map(rho_in):
        # the reference hands the info of the PREVIOUS step to determine_diagtol (self_consistent_field.jl:198-203):
        # its n_iter is 0 and 1 for the first two steps, which therefore both run at diagtol_first
        diagtol = diagtolalg.determine_diagtol(info)
        info["n_iter"] += 1
        t0 = time.time()
        _, ham = energy_hamiltonian(basis, info["psi"], info["occupation"], rho=rho_in,
                                    eigenvalues=info["eigenvalues"], eF=info["eF"], hubbard_n=info["hubbard_n"])
        nxt = next_density(ham, nbandsalg, eigensolver=eigensolver, psi=info["psi"],
                           eigenvalues=info["eigenvalues_global"], occupation=info["occupation_global"], miniter=1,
                           tol=diagtol, generator=gen, fermialg=fermialg)
        info.update(ham=ham, rho_in=rho_in, psi=nxt["psi"], eigenvalues=nxt["eigenvalues"], occupation=nxt["occupation"],
                    eigenvalues_global=nxt["eigenvalues_global"], occupation_global=nxt["occupation_global"],
                    eF=nxt["eF"], rho_out=nxt["rho"], diagonalization=nxt["diagonalization"],
                    n_bands_converge=nxt["n_bands_converge"], n_matvec=info["n_matvec"] + nxt["n_matvec"])
        if hub is not None:
            from .hubbard import compute_hubbard_n
            info["hubbard_n"] = compute_hubbard_n(hub, basis, nxt["psi"], nxt["occupation"])
        if compute_consistent_energies:
            energies = energy(basis, nxt["psi"], nxt["occupation"], rho=nxt["rho"], eigenvalues=nxt["eigenvalues"],
                              eF=nxt["eF"], hubbard_n=info["hubbard_n"])
        else:
            energies = _
        drho = nxt["rho"] - rho_in
        info["energies"] = energies
        info["history_Etot"].append(energies.total)
        info["history_drho"].append(float(drho.norm()) * math.sqrt(basis.dvol))
        nxt_rho = rho_in + mixing.mix_density(basis, drho, rho_in=rho_in, psi=nxt["psi"], eigenvalues=nxt["eigenvalues"],
                                              eF=nxt["eF"], occupation=nxt["occupation"], n_iter=info["n_iter"])
        info["converged"] = basis.comm_kpts.all_true(is_converged(info))
        info["time_step"] = time.time() - t0
        if callback:
            callback(info)
        return nxt_rho

    x = rho
    for _ in range(maxiter):
        fx = fixpoint_map(x)
        if info["converged"]:
            break
        x = acc(x, damping, fx - x)
    rho_f = info["rho_out"]
    energies, ham = energy_hamiltonian(basis, info["psi"], info["occupation"], rho=rho_f,
                                       eigenvalues=info["eigenvalues"], eF=info["eF"], hubbard_n=info["hubbard_n"])
    return dict(ham=ham, basis=basis, energies=energies, converged=info["converged"], rho=rho_f,
                hubbard_n=info["hubbard_n"],
                eigenvalues=info["eigenvalues"], occupation=info["occupation"], eF=info["eF"], psi=info["psi"],
                eigenvalues_global=info["eigenvalues_global"], occupation_global=info["occupation_global"],
                n_iter=info["n_iter"], n_matvec=info["n_matvec"], history_Etot=info["history_Etot"],
                history_drho=info["history_drho"], diagonalization=info["diagonalization"],
                n_bands_converge=info["n_bands_converge"], occupation_threshold=nbandsalg.occupation_threshold,
                runtime_s=time.time() - start, stage="finalize", algorithm="SCF")


def ScfDefaultCallback():
    """scf_callbacks.jl:30-124: the convergence table."""
    def cb(info):
        if info["n_iter"] == 1:
            print("n     Energy            log10(ΔE)   log10(Δρ)   Diag   Δtime")
            print("---   ---------------   ---------   ---------   ----   ------")
        h = info["history_Etot"]
        dE = "" if len(h) < 2 else f"{math.log10(max(abs(h[-1] - h[-2]), 1e-99)):9.2f}"
        diag = np.mean(info["diagonalization"]["n_iter"])
        print(f"{info['n_iter']:3d}   {h[-1]:+15.12f}   {dE:>9}   {math.log10(info['history_drho'][-1]):9.2f}   "
              f"{diag:4.1f}   {info['time_step']:6.2f}s", flush=True)
    return cb
