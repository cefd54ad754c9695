"""Exchange-correlation functionals (oracle; test infrastructure only).

The reference evaluates XC through Libxc.jl (src/DispatchFunctional.jl:55-56,108-128) -- third
party arithmetic that is not under the DFTK.jl tree (Libxc.jl compat "0.3.24", libxc C library
unpinned).  Restated here from the published closed forms with libxc's constants:
  lda_x      Dirac/Slater exchange
  lda_c_vwn  Vosko-Wilk-Nusair 1980 (VWN5, RPA-free fit), libxc lda_c_vwn
  lda_c_pw   Perdew-Wang 1992 (original constants), libxc lda_c_pw
  gga_x_pbe / gga_c_pbe  Perdew-Burke-Ernzerhof 1996 (correlation on PW92 'mod' constants)
Derivatives are obtained with forward-mode dual numbers over NumPy arrays, so that vρ and vσ are
exact derivatives of the same energy expression.  Pinned by test/energies_guess_density.jl:20-36.
"""
import math
import numpy as np


class Dual:
    """Forward-mode AD value with n partial derivatives: d has shape (n,)+v.shape."""
    __slots__ = ("v", "d")
    __array_priority__ = 1000

    def __init__(self, v, d):
        self.v = v
        self.d = d

    @staticmethod
    def lift(x, like):
        if isinstance(x, Dual):
            return x
        return Dual(np.broadcast_to(np.asarray(x, dtype=float), like.v.shape).copy(),
                    np.zeros_like(like.d))

    def __add__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v + o.v, self.d + o.d)
        return Dual(self.v + o, self.d)
    __radd__ = __add__

    def __neg__(self):
        return Dual(-self.v, -self.d)

    def __sub__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v - o.v, self.d - o.d)
        return Dual(self.v - o, self.d)

    def __rsub__(self, o):
        return Dual(o - self.v, -self.d)

    def __mul__(self, o):
        if isinstance(o, Dual):
            return Dual(self.v * o.v, self.d * o.v + o.d * self.v)
        return Dual(self.v * o, self.d * o)
    __rmul__ = __mul__

    def __truediv__(self, o):
        if isinstance(o, Dual):
            q = self.v / o.v
            return Dual(q, (self.d - o.d * q) / o.v)
        return Dual(self.v / o, self.d / o)

    def __rtruediv__(self, o):
        q = o / self.v
        return Dual(q, -self.d * q / self.v)

    def __pow__(self, p):
        return Dual(self.v ** p, self.d * (p * self.v ** (p - 1)))


def _f1(x, f, df):
    if isinstance(x, Dual):
        return Dual(f(x.v), x.d * df(x.v))
    return f(x)


def dlog(x): return _f1(x, np.log, lambda v: 1 / v)
def dexp(x): return _f1(x, np.exp, np.exp)
def dlog1p(x): return _f1(x, np.log1p, lambda v: 1 / (1 + v))
def dexpm1(x): return _f1(x, np.expm1, np.exp)
def dsqrt(x): return _f1(x, np.sqrt, lambda v: 0.5 / np.sqrt(v))
def datan(x): return _f1(x, np.arctan, lambda v: 1 / (1 + v * v))
def dcbrt(x): return _f1(x, np.cbrt, lambda v: np.cbrt(v) / (3 * v))


# ------------------------------------------------------------------ LDA pieces
_RS_FAC = (3 / (4 * math.pi)) ** (1 / 3)
_FZ_DEN = 2 ** (4 / 3) - 2
_FPP0 = 4 / (9 * (2 ** (1 / 3) - 1))


# libxc's edge semantics (restated from its documented behaviour; the values are not checked against libxc's sources
# in this tree): a point with total density at or below DENS_THRESHOLD is zero; a spin channel at or below
# DENS_THRESHOLD_SPIN contributes nothing to spin-resolved exchange; (1 +- zeta)^p at or below ZETA_THRESHOLD
# (DBL_EPSILON) is frozen there with zero derivative; sigma_uu, sigma_dd are raised to SIGMA_FLOOR, the square of
# the sigma threshold 1e-15^(4/3), with derivatives taken at the raised value.  A negative spin density is raised to
# zero before zeta is formed (derivatives taken there), so that |zeta| <= 1; libxc is recalled to raise it to the
# density threshold instead, which is not adopted (see xc_core.cuh).
DENS_THRESHOLD = 1e-15
DENS_THRESHOLD_SPIN = 1e-15
ZETA_THRESHOLD = 2.220446049250313e-16
SIGMA_FLOOR = 1e-40


def _opz_pow(opz, p):
    """(1 + zeta)^p given opz = 1 + zeta, frozen below the zeta threshold."""
    frozen = opz.v <= ZETA_THRESHOLD
    x = np.where(frozen, 1.0, opz.v)
    return Dual(np.where(frozen, ZETA_THRESHOLD ** p, x ** p),
                np.where(frozen, 0.0, opz.d * (p * x ** (p - 1))))


def _fzeta(spin):
    _, opz, omz = spin
    return (_opz_pow(opz, 4 / 3) + _opz_pow(omz, 4 / 3) - 2) / _FZ_DEN


def _ex_unif_unpol(rho):
    """ε_x ρ for spin-unpolarised density."""
    return -(3 / 4) * (3 / math.pi) ** (1 / 3) * rho * dcbrt(rho)


def _vwn_piece(x, A, b, c, x0):
    Q = math.sqrt(4 * c - b * b)
    X = x * x + b * x + c
    X0 = x0 * x0 + b * x0 + c
    at = datan(Q / (2 * x + b))
    return A * (dlog(x * x / X) + (2 * b / Q) * at
                - (b * x0 / X0) * (dlog((x - x0) * (x - x0) / X) + (2 * (b + 2 * x0) / Q) * at))


_VWN = dict(A=(0.0310907, 0.01554535, -1 / (6 * math.pi ** 2)),
            b=(3.72744, 7.06042, 1.13107), c=(12.9352, 18.0578, 13.0045),
            x0=(-0.10498, -0.32500, -0.0047584))


def _ec_vwn(rs, spin):
    x = dsqrt(rs)
    p = [_vwn_piece(x, _VWN["A"][i], _VWN["b"][i], _VWN["c"][i], _VWN["x0"][i]) for i in range(3)]
    if spin is None:
        return p[0]
    fz = _fzeta(spin)
    z4 = spin[0] ** 4
    return p[0] + p[2] * fz * (1 - z4) / _FPP0 + (p[1] - p[0]) * fz * z4


_PW = dict(a=(0.0310907, 0.01554535, 0.0168869), fz20=1.709921)
_PWMOD = dict(a=(0.0310906908696548950, 0.01554534543482744750, 0.0168868639404617),
              fz20=1.709920934161365617563962776245)
_PW_COMMON = dict(a1=(0.21370, 0.20548, 0.11125), b1=(7.5957, 14.1189, 10.357),
                  b2=(3.5876, 6.1977, 3.6231), b3=(1.6382, 3.3662, 0.88026),
                  b4=(0.49294, 0.62517, 0.49671))


def _pw_G(rs, i, par):
    a = par["a"][i]
    c = _PW_COMMON
    srs = dsqrt(rs)
    den = 2 * a * (c["b1"][i] * srs + c["b2"][i] * rs + c["b3"][i] * rs * srs + c["b4"][i] * rs * rs)
    return -2 * a * (1 + c["a1"][i] * rs) * dlog1p(1 / den)


def _ec_pw(rs, spin, par):
    g0 = _pw_G(rs, 0, par)
    if spin is None:
        return g0
    g1 = _pw_G(rs, 1, par)
    mac = _pw_G(rs, 2, par)  # this is -alpha_c
    fz = _fzeta(spin)
    z4 = spin[0] ** 4
    return g0 - mac * fz * (1 - z4) / par["fz20"] + (g1 - g0) * fz * z4


# ------------------------------------------------------------------ PBE pieces
_KAPPA = 0.8040
_BETA = 0.06672455060314922
_MU = _BETA * (math.pi ** 2 / 3)
_GAMMA = (1 - math.log(2)) / math.pi ** 2


def _ex_pbe_unpol(rho, sigma):
    kF = dcbrt(3 * math.pi ** 2 * rho)
    s2 = sigma / (4 * kF * kF * rho * rho)
    Fx = 1 + _KAPPA - _KAPPA / (1 + _MU * s2 / _KAPPA)
    return _ex_unif_unpol(rho) * Fx


def _ec_pbe(rho, rs, spin, sigma_tot):
    ec = _ec_pw(rs, spin, _PWMOD)
    if spin is None:
        phi = 1.0
        phi3 = 1.0
    else:
        phi = (_opz_pow(spin[1], 2 / 3) + _opz_pow(spin[2], 2 / 3)) / 2
        phi3 = phi * phi * phi
    kF = dcbrt(3 * math.pi ** 2 * rho)
    ks2 = 4 * kF / math.pi
    t2 = sigma_tot / (4 * (phi * phi) * ks2 * rho * rho)
    A = (_BETA / _GAMMA) / dexpm1(-ec / (_GAMMA * phi3))
    At2 = A * t2
    H = _GAMMA * phi3 * dlog1p((_BETA / _GAMMA) * t2 * (1 + At2) / (1 + At2 + At2 * At2))
    return ec + H


# ------------------------------------------------------------------ driver
def evaluate(functionals, rho, sigma=None):
    """rho: (n_spin, N) array; sigma: None (LDA) or (n_sigma, N) with n_sigma = 1 (unpolarised)
    or 3 (uu, ud, dd).  Returns dict(e=(N,), Vrho=(n_spin,N), Vsigma=(n_sigma,N) or None), the
    same quantities libxc returns as zk*rho, vrho, vsigma (cf. xc.jl:104-113)."""
    n_spin, N = rho.shape
    is_gga = any(f.startswith("gga") for f in functionals)
    if is_gga:
        assert sigma is not None
    nvar = n_spin + (sigma.shape[0] if is_gga else 0)
    rho_tot = rho.sum(axis=0)
    mask = rho_tot > DENS_THRESHOLD
    safe = np.where(mask, rho, 1.0 / n_spin)

    def var(i, val):
        d = np.zeros((nvar, N))
        d[i] = 1.0
        return Dual(val.copy(), d)

    r = [var(s, np.maximum(safe[s], 0.0)) for s in range(n_spin)]
    sg = None
    if is_gga:
        ssafe = np.where(mask, sigma, 0.0)
        floored = [0] if sigma.shape[0] == 1 else [0, 2]      # sigma_ud is not floored
        ssafe[floored] = np.maximum(ssafe[floored], SIGMA_FLOOR)
        sg = [var(n_spin + i, ssafe[i]) for i in range(sigma.shape[0])]
    if n_spin == 1:
        n = r[0]
        spin = None
    else:
        n = r[0] + r[1]
        # zeta and 1 +- zeta = 2 rho_s / n, which keep their relative precision as zeta -> +-1
        spin = ((r[0] - r[1]) / n, 2 * r[0] / n, 2 * r[1] / n)
    rs = _RS_FAC / dcbrt(n)

    def screened(s, piece):
        """A spin channel's exchange, zero (value and derivatives) at or below the channel threshold."""
        live = r[s].v > DENS_THRESHOLD_SPIN
        x = piece(Dual(np.where(live, r[s].v, 1.0), r[s].d))
        return Dual(np.where(live, x.v, 0.0), np.where(live[None, :], x.d, 0.0))
    e = Dual(np.zeros(N), np.zeros((nvar, N)))
    for f in functionals:
        if f == "lda_x":
            if n_spin == 1:
                e = e + _ex_unif_unpol(n)
            else:
                for s in range(2):
                    e = e + screened(s, lambda rr: 0.5 * _ex_unif_unpol(2 * rr))
        elif f == "lda_c_vwn":
            e = e + n * _ec_vwn(rs, spin)
        elif f == "lda_c_pw":
            e = e + n * _ec_pw(rs, spin, _PW)
        elif f == "gga_x_pbe":
            if n_spin == 1:
                e = e + _ex_pbe_unpol(n, sg[0])
            else:
                for s, isg in ((0, 0), (1, 2)):
                    e = e + screened(s, lambda rr: 0.5 * _ex_pbe_unpol(2 * rr, 4 * sg[isg]))
        elif f == "gga_c_pbe":
            stot = sg[0] if n_spin == 1 else sg[0] + 2 * sg[1] + sg[2]
            e = e + n * _ec_pbe(n, rs, spin, stot)
        else:
            raise NotImplementedError(f)
    ev = np.where(mask, e.v, 0.0)
    dv = np.where(mask[None, :], e.d, 0.0)
    return dict(e=ev, Vrho=dv[:n_spin], Vsigma=dv[n_spin:] if is_gga else None)
