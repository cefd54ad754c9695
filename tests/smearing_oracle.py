"""Oracle for the non-monotone smearings, the two-stage Fermi-level search and energy-cutoff smearing (test
infrastructure only): a NumPy restatement of src/Smearing.jl:118-168, src/occupation.jl:18-21,138-155 and
src/terms/kinetic.jl:63-110 that never imports the product, plus `extended()`, which runs the oracle of `oracle/`
(SCF, energies, Hψ) with these pieces in place of its Fermi-Dirac/Gaussian-only occupation and its |p|²/2 kinetic
table.  The Hermite polynomials come from numpy.polynomial.hermite (physicists' convention), the derivatives from
differentiating the series term by term."""
import contextlib
import math
import numpy as np
from numpy.polynomial import hermite as npherm
from scipy.special import erf, erfc

import oracle.scf as _oscf
import oracle.terms as _oterms

_EPS = np.finfo(float).eps
_BASE_COMPUTE_OCCUPATION = _oscf.compute_occupation


def _mp(kind):
    if isinstance(kind, (tuple, list)) and kind[0] == "MethfesselPaxton":
        return int(kind[1])
    return None


def _A(i):
    return (-1) ** i / (math.factorial(i) * 4 ** i * math.sqrt(math.pi))


def _herm(x, k):
    c = np.zeros(k + 1)
    c[k] = 1.0
    return npherm.hermval(x, c)


def occupation(kind, x):
    x = np.asarray(x, dtype=float)
    n = _mp(kind)
    if kind == "MarzariVanderbilt":
        y = -x - 1 / math.sqrt(2)
        return -erf(x + 1 / math.sqrt(2)) / 2 + np.exp(-y * y) / math.sqrt(2 * math.pi) + 0.5
    if n is not None:
        out = np.empty_like(x)
        inf = np.isinf(x)
        out[inf] = (x[inf] < 0).astype(float)
        xf = x[~inf]
        out[~inf] = erfc(xf) / 2 + np.exp(-xf * xf) * sum((_A(i) * _herm(xf, 2 * i - 1) for i in range(1, n + 1)),
                                                          np.zeros_like(xf))
        return out
    return _oterms.smearing_occupation(kind, x)


def entropy(kind, x):
    x = np.asarray(x, dtype=float)
    n = _mp(kind)
    if kind == "MarzariVanderbilt":
        y = x + 1 / math.sqrt(2)
        return y * np.exp(-y * y) / math.sqrt(2 * math.pi)
    if n is not None:
        return np.exp(-x * x) * sum(_A(i) * (_herm(x, 2 * i) / 2 + (2 * i * _herm(x, 2 * i - 2) if i > 0 else 0.0))
                                    for i in range(n + 1))
    return _oterms.smearing_entropy(kind, x)


def occupation_derivative(kind, x):
    """f'(x) by differentiating each smearing's formula (product rule on the Hermite series)."""
    x = np.asarray(x, dtype=float)
    n = _mp(kind)
    if kind == "None":
        return np.zeros_like(x)
    if kind == "FermiDirac":
        f = _oterms.smearing_occupation(kind, x)
        return -f * (1 - f)
    if kind == "Gaussian":
        return -np.exp(-x * x) / math.sqrt(math.pi)
    if kind == "MarzariVanderbilt":
        y = x + 1 / math.sqrt(2)
        return -np.exp(-y * y) / math.sqrt(math.pi) - 2 * y * np.exp(-y * y) / math.sqrt(2 * math.pi)
    if n is not None:
        g = np.exp(-x * x)
        d = -g / math.sqrt(math.pi)
        for i in range(1, n + 1):
            c = np.zeros(2 * i)
            c[2 * i - 1] = _A(i)
            d = d + g * (npherm.hermval(x, npherm.hermder(c)) - 2 * x * npherm.hermval(x, c))
        return d
    raise NotImplementedError(kind)


# ------------------------------------------------------------------ blow-ups, kinetic.jl:63-110
def blowup_chv(p, Ecut):
    out = np.ones_like(np.asarray(p, dtype=float))
    for i, y in enumerate(np.asarray(p, dtype=float).ravel()):
        x = y / math.sqrt(2 * Ecut)
        if x < 0.85:
            continue
        blow = 0.013952310177257383 / (1 - x) ** 2
        ratio = Ecut / (y * y / 2)
        if x < 0.90:
            f = lambda t: 0.0 if t == 0 else math.exp(-1 / t)
            t = (x - 0.85) / (0.90 - 0.85)
            s = f(t) / (f(t) + f(1 - t))
            out.flat[i] = ratio * ((1 - s) * x * x + s * blow)
        else:
            out.flat[i] = ratio * blow
    return out


def blowup_abinit(p, Ecut, Ecutsm=0.5):
    Es = Ecut * Ecutsm
    assert Es < Ecut
    out = np.ones_like(np.asarray(p, dtype=float))
    for i, y in enumerate(np.asarray(p, dtype=float).ravel()):
        if y > math.sqrt(2 * (Ecut - Es)):
            x = (Ecut - y * y / 2) / Es
            out.flat[i] = 1 / (x * x * (3 + x - 6 * x * x + 3 * x * x))
    return out


BLOWUPS = {"CHV": blowup_chv, "Abinit": blowup_abinit}


# ------------------------------------------------------------------ Fermi level, occupation.jl:18-21,103-155
def _roots_secant_bisection(f, x):
    """Roots.find_zero(f, x, Secant(), Bisection(); atol=eps), written out as the hybrid iterates its state
    (xn0, xn1, fxn0, fxn1)."""
    h = _EPS ** (1 / 3)
    xn1 = float(x)
    xn0 = xn1 + h + abs(xn1) * h ** 2
    fxn0, fxn1 = f(xn0), f(xn1)

    def bisection(a, b):
        fa = f(a)
        for _ in range(2000):
            m = a + (b - a) / 2
            if m in (a, b):
                break
            fm = f(m)
            if fm == 0:
                return m
            if np.sign(fm) == np.sign(fa):
                a, fa = m, fm
            else:
                b = m
        return a + (b - a) / 2

    quad = 0
    for _ in range(1000):
        if abs(fxn1) <= max(_EPS, 4 * _EPS * abs(xn1)):
            return xn1
        if abs(xn1 - xn0) <= max(_EPS, _EPS * max(abs(xn1), abs(xn0))):
            return xn1
        step = fxn1 * (xn1 - xn0) / (fxn1 - fxn0)
        if not np.isfinite(step) or step == 0:
            return xn1
        p0, p1, q0, q1 = xn1, xn1 - step, fxn1, None
        q1 = f(p1)
        if q1 == 0:
            return p1
        if np.sign(q0) * np.sign(q1) < 0:
            return bisection(p0, p1)
        adjusted = False
        if abs(p1 - xn1) >= 100 * abs(xn1 - xn0):
            adjusted, p1 = True, xn1 + np.sign(p1 - xn1) * 100 * abs(xn1 - xn0)
            q1 = f(p1)
        elif abs(p1 - xn1) <= abs(xn1 - xn0) / 1000:
            adjusted, p1 = True, xn1 + np.sign(p1 - xn1) * abs(xn1 - xn0) / 1000
            q1 = f(p1)
        if np.sign(fxn1) * np.sign(q1) < 0:
            return bisection(xn1, p1)
        if adjusted or abs(q1) < abs(fxn1):
            xn0, fxn0, xn1, fxn1 = p0, q0, p1, q1
            quad = 0
            continue
        if quad > 4:
            return p1
        quad += 1
        a, fa, b, fb, c, fc = xn0, fxn0, xn1, fxn1, p1, q1
        fba, fbc = (fb - fa) / (b - a), (fb - fc) / (b - c)
        r = 0.5 * ((a + b) - fba / (fbc - fba) * (c - a))
        if np.isfinite(r):
            xn0, fxn0, xn1, fxn1 = p0, q0, r, f(r)
        else:
            xn0, fxn0, xn1, fxn1 = p0, q0, p1, q1
    return xn1


def _excess(model, weights, eigenvalues, eF, smearing):
    n = sum(w * model.filled_occupation * occupation(smearing, (e - eF) / model.temperature).sum()
            for w, e in zip(weights, eigenvalues))
    return n - model.n_electrons


def _bisection_level(model, weights, eigenvalues, tol_n_elec, smearing):
    n_fill = -(-model.n_electrons // (model.n_spin_components * model.filled_occupation))
    homo = max(e[n_fill - 1] for e in eigenvalues)
    lumo = [e[n_fill:].min() for e in eigenvalues if len(e) > n_fill]
    eF = (homo + min(lumo)) / 2 if lumo else homo + 1
    ex = _excess(model, weights, eigenvalues, eF, smearing)
    if abs(ex) < tol_n_elec / 10:
        return eF
    lo, hi = (eF, max(e.max() for e in eigenvalues) + 1) if ex < 0 else (min(e.min() for e in eigenvalues) - 1, eF)
    while True:
        mid = (lo + hi) / 2
        if mid in (lo, hi):
            return mid
        if _excess(model, weights, eigenvalues, mid, smearing) < 0:
            lo = mid
        else:
            hi = mid


def fermi_level(model, weights, eigenvalues, fermialg=None, tol_n_elec=1e-6):
    """εF of the oracle: bisection for None/FermiDirac/Gaussian (default_fermialg), else the two-stage search."""
    eigenvalues = [np.asarray(e, dtype=float) for e in eigenvalues]
    if fermialg is None:
        fermialg = "bisection" if model.smearing in ("None", "FermiDirac", "Gaussian") else "two-stage"
    if fermialg == "bisection":
        return _bisection_level(model, weights, eigenvalues, tol_n_elec, model.smearing)
    guess = _bisection_level(model, weights, eigenvalues, tol_n_elec, "Gaussian")
    return _roots_secant_bisection(lambda x: _excess(model, weights, eigenvalues, x, model.smearing), guess)


def compute_occupation(basis, eigenvalues, tol_n_elec=1e-6):
    """Drop-in for oracle.scf.compute_occupation with every smearing."""
    m = basis.model
    if m.temperature == 0:
        return _BASE_COMPUTE_OCCUPATION(basis, eigenvalues, tol_n_elec=tol_n_elec)
    eF = fermi_level(m, basis.kweights, eigenvalues, tol_n_elec=tol_n_elec)
    return [m.filled_occupation * occupation(m.smearing, (np.asarray(e) - eF) / m.temperature)
            for e in eigenvalues], eF


@contextlib.contextmanager
def extended(blowup=None):
    """Run the oracle (oracle.scf / oracle.terms) with every smearing and, if `blowup` is "CHV" or "Abinit", the
    blown-up kinetic table |p|²/2 · blowup(|p|, Ecut)."""
    saved = (_oscf.compute_occupation, _oterms.smearing_entropy, _oterms.kinetic_energies)
    base_kinetic = _oterms.kinetic_energies

    def kinetic_energies(basis, kpt):
        p = basis.Gplusk_cart(kpt)
        return base_kinetic(basis, kpt) * BLOWUPS[blowup](np.linalg.norm(p, axis=1), basis.Ecut)

    _oscf.compute_occupation = compute_occupation
    _oterms.smearing_entropy = entropy
    if blowup is not None:
        _oterms.kinetic_energies = kinetic_energies
    try:
        yield
    finally:
        _oscf.compute_occupation, _oterms.smearing_entropy, _oterms.kinetic_energies = saved
