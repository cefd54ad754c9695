"""Fermi level and occupations (mirror of src/occupation.jl).  The reference performs one scalar
allreduce per bisection step (occupation.jl:23-27); here all eigenvalues are allgathered once and the
Fermi-level search runs redundantly on every rank, which yields a bit-identical Fermi level everywhere."""
import math
import numpy as np
from .terms import smearing_occupation, occupation_derivative


def gather_eigenvalues(basis, eigenvalues, stats=()):
    """ONE fixed-size allgather per SCF step: the eigenvalues of every rank's blocks (all blocks carry the same number
    of bands) with a few per-rank solver statistics behind them.  Returns (eigenvalues of all blocks in global block
    order b = ik + spin * n_kpt, their k-weights, stats[rank, :])."""
    comm = basis.comm_kpts
    layout = getattr(basis, "layout", None)
    stats = np.asarray(stats, dtype=np.float64).reshape(-1)
    if comm.nranks == 1:
        w = list(layout.weights) if layout is not None else list(basis.kweights)
        return [np.asarray(e, dtype=np.float64) for e in eigenvalues], w, stats[None, :]
    nb = len(eigenvalues[0])
    if any(len(e) != nb for e in eigenvalues):
        raise ValueError("all blocks must carry the same number of bands")
    buf = np.zeros(layout.max_local * nb + len(stats))
    for j, e in enumerate(eigenvalues):
        buf[j * nb:(j + 1) * nb] = e
    buf[layout.max_local * nb:] = stats
    got = comm.allgather(buf)
    ev = [None] * layout.n_blocks
    for r in range(comm.nranks):
        for j, b in enumerate(layout.blocks_of_rank[r]):
            ev[b] = got[r, j * nb:(j + 1) * nb].copy()
    return ev, list(layout.weights), got[:, layout.max_local * nb:]


def _occ(model, eigs, eF, smearing=None):
    if model.temperature == 0:
        return [model.filled_occupation * smearing_occupation("None", e - eF) for e in eigs]
    smearing = model.smearing if smearing is None else smearing
    return [model.filled_occupation * smearing_occupation(smearing, (e - eF) / model.temperature) for e in eigs]


class _FermiSearch:
    """The electron-count equation over ONE flat array of all eigenvalues of all blocks with their k-weights: an
    evaluation is one vectorised pass (a search needs ~60 of them; a per-block Python loop over 84 blocks made this a
    third of a metal's SCF step)."""

    def __init__(self, model, ev, w, eF_int, tol_n_elec):
        self.model, self.eF_int, self.tol_n_elec = model, eF_int, tol_n_elec
        self.e_all = np.concatenate([np.asarray(e, dtype=np.float64) for e in ev])
        self.w_all = np.concatenate([np.full(len(e), float(wk)) for wk, e in zip(w, ev)])
        self.e_min, self.e_max = min(e.min() for e in ev), max(e.max() for e in ev)

    def excess(self, eF, smearing=None):
        return float(np.dot(self.w_all, _occ(self.model, [self.e_all], eF, smearing)[0])) - self.model.n_electrons

    def dexcess(self, eF):
        """d excess / d εF from the closed-form occupation derivative."""
        m = self.model
        fp = occupation_derivative(m.smearing, (self.e_all - eF) / m.temperature)
        return -m.filled_occupation * float(np.dot(self.w_all, fp)) / m.temperature


class FermiBisection:
    """occupation.jl:103-137: bisection of the electron count, for monotone smearing functions."""

    def fermi_level(self, search, smearing=None):
        def excess(eF):
            return search.excess(eF, smearing)
        eF = search.eF_int
        ex = excess(eF)
        if abs(ex) >= search.tol_n_elec / 10:
            lo, hi = (eF, search.e_max + 1) if ex < 0 else (search.e_min - 1, eF)
            if not (excess(lo) <= 0 <= excess(hi)):      # occupation.jl:100-103 (@assert on the bracket)
                raise RuntimeError("compute_occupation: the Fermi level is not bracketed by the eigenvalue range")
            eF = _bisect(excess, lo, hi)
        return eF

    def __repr__(self):
        return "FermiBisection()"


class FermiTwoStage:
    """occupation.jl:138-155: a Gaussian-smearing bisection, then the root of the real smearing's electron count
    nearest to it (secant from that guess, bisection once a sign change brackets a root).  For the non-monotone
    Marzari-Vanderbilt and Methfessel-Paxton smearings, whose electron count can have several roots."""

    def fermi_level(self, search, smearing=None):
        eF = FermiBisection().fermi_level(search, "Gaussian")
        return find_zero_secant_bisection(lambda x: search.excess(x, smearing), eF)

    def __repr__(self):
        return "FermiTwoStage()"


def default_fermialg(smearing):
    """occupation.jl:18-21: bisection for the monotone smearings, the two-stage search for the others."""
    return FermiBisection() if smearing in ("None", "FermiDirac", "Gaussian") else FermiTwoStage()


def _bisect(f, lo, hi):
    """Roots.Bisection to atol = eps on a bracket with f(lo) <= 0 <= f(hi)."""
    for _ in range(200):
        mid = (lo + hi) / 2
        if mid == lo or mid == hi:
            break
        if f(mid) < 0:
            lo = mid
        else:
            hi = mid
    return (lo + hi) / 2


def _bisect_bracket(f, a, fa, b, fb):
    """Bisection on a bracket (a, b) with f(a) f(b) < 0 in either orientation."""
    if fa > 0:
        a, b = b, a
    return _bisect(f, a, b)


def find_zero_secant_bisection(f, x, atol=np.finfo(float).eps, maxiters=1000):
    """Roots.find_zero(f, x, Secant(), Bisection(); atol): secant steps from x (the second start point is
    x + cbrt(eps) + |x| cbrt(eps)²) with the hybrid's guards -- a step longer than 100 or shorter than 1/1000 of the
    previous one is clamped to that length, a step that does not reduce |f| is replaced by the vertex of the parabola
    through the last three points (at most 5 times in a row) -- and bisection on the first pair of consecutive
    points whose values change sign.  Converged when |f| <= max(atol, 4 eps |x|) or two points agree to eps."""
    eps = np.finfo(float).eps
    h = eps ** (1 / 3)
    x0, x1 = x + (h + abs(x) * h * h), float(x)
    f0, f1 = f(x0), f(x1)
    quad_ctr = 0
    for _ in range(maxiters):
        if not (math.isfinite(x1) and math.isfinite(f1)):
            break
        if abs(f1) <= max(atol, 4 * eps * abs(x1)) or abs(x1 - x0) <= eps * max(1.0, abs(x1), abs(x0)):
            break
        den = f1 - f0
        delta = f1 * (x1 - x0) / den if den != 0 else math.inf
        if delta == 0 or not math.isfinite(delta):
            break
        r = x1 - delta
        fr = f(r)
        if fr == 0:
            return r
        if np.sign(f1) * np.sign(fr) < 0:
            return _bisect_bracket(f, x1, f1, r, fr)
        adj = False
        dr, dx = abs(r - x1), abs(x1 - x0)
        if dr >= 100 * dx:
            adj, r = True, x1 + math.copysign(100 * dx, r - x1)
            fr = f(r)
        elif dr <= dx / 1000:
            adj, r = True, x1 + math.copysign(dx / 1000, r - x1)
            fr = f(r)
        if np.sign(f1) * np.sign(fr) < 0:
            return _bisect_bracket(f, x1, f1, r, fr)
        if adj or abs(fr) < abs(f1):
            x0, f0, x1, f1 = x1, f1, r, fr
            quad_ctr = 0
            continue
        if quad_ctr > 4:
            x0, f0, x1, f1 = x1, f1, r, fr
            break
        quad_ctr += 1
        # vertex of the parabola through (r, fr), (x1, f1), (x0, f0) (Roots.quad_vertex)
        fba = (f1 - f0) / (x1 - x0)
        fbc = (f1 - fr) / (x1 - r)
        q = 0.5 * ((x0 + x1) - fba / (fbc - fba) * (r - x0))
        if math.isfinite(q):
            x0, f0, x1, f1 = x1, f1, q, f(q)
        else:
            x0, f0, x1, f1 = x1, f1, r, fr
    return x1


def compute_occupation(basis, eigenvalues, *, fermialg=None, tol_n_elec=1e-6, gathered=None, return_global=False,
                       eF=None):
    """Returns (occupation of the local blocks, εF).  `fermialg`: FermiBisection() or FermiTwoStage() (default:
    default_fermialg(model.smearing)).  `gathered` = (eigenvalues of all blocks, weights) when the caller already did
    the allgather (next_density packs solver statistics into the same collective).  `eF` given: the occupations at that
    Fermi level, without a search (occupation.jl, compute_occupation(basis, eigenvalues, εF))."""
    model = basis.model
    for ek in eigenvalues:
        if not np.all(np.diff(ek) >= -np.finfo(float).eps):
            raise ValueError("Eigenvalues should be monotonically increasing.")
    if eF is not None:
        occ = _occ(model, [np.asarray(e) for e in eigenvalues], eF)
        if not return_global:
            return occ, eF
        ev = gathered[0] if gathered is not None else gather_eigenvalues(basis, eigenvalues)[0]
        return occ, eF, _occ(model, ev, eF)
    ev, w = gathered if gathered is not None else gather_eigenvalues(basis, eigenvalues)[:2]
    filled = model.filled_occupation
    if model.n_electrons == 0:
        eF = min(e.min() for e in ev) - 1.0
        occ = [np.zeros(len(e)) for e in eigenvalues]
        return (occ, eF, [np.zeros(len(e)) for e in ev]) if return_global else (occ, eF)

    if filled * sum(wk * len(e) for wk, e in zip(w, ev)) < model.n_electrons - tol_n_elec:
        raise RuntimeError("Could not obtain required number of electrons by filling every state. Increase n_bands.")
    n_fill = -(-model.n_electrons // (model.n_spin_components * filled))
    HOMO = max(e[n_fill - 1] for e in ev)
    lum = [e[n_fill:].min() for e in ev if len(e) > n_fill]
    eF = (HOMO + min(lum)) / 2 if lum else HOMO + 1
    search = _FermiSearch(model, ev, w, eF, tol_n_elec)
    if model.temperature == 0:
        if model.n_electrons % (model.n_spin_components * filled) != 0:
            raise RuntimeError(f"{model.n_electrons} electrons cannot be attained by filling states with "
                               f"occupation {filled}; add a temperature or use collinear spin")
        if abs(search.excess(eF)) > tol_n_elec:
            raise RuntimeError("Unable to find non-fractional occupations that have the correct number of "
                               "electrons. You should add a temperature.")
    else:
        fermialg = default_fermialg(model.smearing) if fermialg is None else fermialg
        eF = fermialg.fermi_level(search)
        import warnings           # occupation.jl:72-99
        if abs(search.excess(eF)) > tol_n_elec:
            warnings.warn("Large deviation of electron count in compute_occupation. This may lead to an unphysical "
                          "solution. Try decreasing the temperature or using a different smearing function.")
        if search.dexcess(eF) < -math.sqrt(np.finfo(float).eps):
            warnings.warn("Negative density of states (electron count versus Fermi level derivative) encountered in "
                          "compute_occupation. This may lead to an unphysical solution. Try decreasing the "
                          "temperature or using a different smearing function.")
    occ = _occ(model, [np.asarray(e) for e in eigenvalues], eF)
    return (occ, eF, _occ(model, ev, eF)) if return_global else (occ, eF)
