"""Extended-precision reference for the exchange-correlation functionals the XC kernel carries (test infrastructure).

The five functionals are restated from the papers' closed forms with libxc's constants, in mpmath at `DPS` digits:
  lda_x      Dirac exchange, e = -(3/4) (3/pi)^(1/3) n^(4/3); spin-resolved as (e[2 rho_up] + e[2 rho_dn]) / 2
  lda_c_vwn  Vosko, Wilk, Nusair, Can. J. Phys. 58, 1200 (1980), parametrisation 5 with the spin-stiffness fit
  lda_c_pw   Perdew, Wang, Phys. Rev. B 45, 13244 (1992)
  gga_x_pbe  Perdew, Burke, Ernzerhof, Phys. Rev. Lett. 77, 3865 (1996), exchange enhancement factor
  gga_c_pbe  the same paper's gradient correction H on PW92 with the "modified" constants (A = gamma, gamma / 2,
             1 / (6 pi^2) and f''(0) from its closed form)
vrho and vsigma are not restated: they are central finite differences of the energy density at `DPS` digits
(mpmath.diff with a step 1e-25 relative to the variable), so they check a kernel's derivatives without sharing its
derivative arithmetic.

libxc, which the reference program calls, evaluates these functionals with some edge semantics, restated here as
named parameters.  Their values are recalled from libxc's documented behaviour and are NOT checked against libxc's
sources (which are not part of this project); the tests built on them depend on the behaviour on each side of a
threshold, not on its exact value:
  DENS_THRESHOLD       a point whose total density is at or below it gives zero energy and potentials;
  DENS_THRESHOLD_SPIN  a spin channel at or below it contributes nothing to spin-resolved exchange;
  ZETA_THRESHOLD       (1 +- zeta)^p with 1 +- zeta at or below it is frozen at ZETA_THRESHOLD^p, zero derivative;
  SIGMA_FLOOR          sigma_uu, sigma_dd (the unpolarised sigma) are raised to it, derivatives taken there.
A negative spin density is raised to zero, derivatives taken there, so that |zeta| <= 1.  libxc is recalled to raise
each spin density to the functional's density threshold instead; that floor is not restated (nor checked).
"""
import mpmath as mp

DPS = 50
DENS_THRESHOLD = 1e-15
DENS_THRESHOLD_SPIN = 1e-15
ZETA_THRESHOLD = 2.220446049250313e-16   # DBL_EPSILON
SIGMA_FLOOR = 1e-40                      # (1e-15^(4/3))^2

FUNCTIONALS = ("lda_x", "lda_c_vwn", "lda_c_pw", "gga_x_pbe", "gga_c_pbe")

_VWN_PARAMS = (   # (A, b, c, x0): paramagnetic, ferromagnetic, spin stiffness
    ("0.0310907", "3.72744", "12.9352", "-0.10498"),
    ("0.01554535", "7.06042", "18.0578", "-0.32500"),
    (None, "1.13107", "13.0045", "-0.0047584"),          # A = -1 / (6 pi^2)
)
_PW_FIT = (   # (alpha1, beta1, beta2, beta3, beta4): paramagnetic, ferromagnetic, -alpha_c
    ("0.21370", "7.5957", "3.5876", "1.6382", "0.49294"),
    ("0.20548", "14.1189", "6.1977", "3.3662", "0.62517"),
    ("0.11125", "10.357", "3.6231", "0.88026", "0.49671"),
)
_PW_A = ("0.0310907", "0.01554535", "0.0168869")
_PW_FZ20 = "1.709921"
KAPPA = "0.804"
BETA = "0.06672455060314922"


def _mpf(x):
    return mp.mpf(x)


def _gamma():
    return (1 - mp.log(2)) / mp.pi ** 2


def _opz_pow(x, p):
    """(1 + zeta)^p at x = 1 + zeta, frozen at the zeta threshold."""
    thr = _mpf(ZETA_THRESHOLD)
    return thr ** p if x <= thr else x ** p


def _f_zeta(opz, omz):
    return (_opz_pow(opz, mp.mpf(4) / 3) + _opz_pow(omz, mp.mpf(4) / 3) - 2) / (mp.cbrt(2) * 2 - 2)


def _fpp0():
    return mp.mpf(8) / 9 / (2 * mp.cbrt(2) - 2)


def ex_lda(n):
    """Dirac exchange energy per volume of an unpolarised density n."""
    return -mp.mpf(3) / 4 * mp.cbrt(3 / mp.pi) * n * mp.cbrt(n)


def _vwn(rs, i):
    A, b, c, x0 = _VWN_PARAMS[i]
    A = -1 / (6 * mp.pi ** 2) if A is None else _mpf(A)
    b, c, x0 = _mpf(b), _mpf(c), _mpf(x0)
    x = mp.sqrt(rs)
    X = x * x + b * x + c
    X0 = x0 * x0 + b * x0 + c
    Q = mp.sqrt(4 * c - b * b)
    at = mp.atan(Q / (2 * x + b))
    return A * (mp.log(x * x / X) + 2 * b / Q * at
                - b * x0 / X0 * (mp.log((x - x0) ** 2 / X) + 2 * (b + 2 * x0) / Q * at))


def _pw_g(rs, i, A):
    a1, b1, b2, b3, b4 = (_mpf(v) for v in _PW_FIT[i])
    den = 2 * A * (b1 * mp.sqrt(rs) + b2 * rs + b3 * rs ** mp.mpf(1.5) + b4 * rs ** 2)
    return -2 * A * (1 + a1 * rs) * mp.log(1 + 1 / den)


def eps_c_lda(rs, spin, kind):
    """Correlation energy per particle.  spin = None (unpolarised) or (zeta, 1 + zeta, 1 - zeta)."""
    if kind == "vwn":
        e0 = _vwn(rs, 0)
        if spin is None:
            return e0
        z, opz, omz = spin
        f = _f_zeta(opz, omz)
        return e0 + _vwn(rs, 2) * f * (1 - z ** 4) / _fpp0() + (_vwn(rs, 1) - e0) * f * z ** 4
    if kind == "pw":
        As, fz20 = [_mpf(a) for a in _PW_A], _mpf(_PW_FZ20)
    else:   # "pw_mod"
        g = _gamma()
        As, fz20 = [g, g / 2, 1 / (6 * mp.pi ** 2)], _fpp0()
    e0 = _pw_g(rs, 0, As[0])
    if spin is None:
        return e0
    z, opz, omz = spin
    f = _f_zeta(opz, omz)
    alpha_c = -_pw_g(rs, 2, As[2])
    return e0 + alpha_c * f * (1 - z ** 4) / fz20 + (_pw_g(rs, 1, As[1]) - e0) * f * z ** 4


def pbe_fx(s2):
    kappa = _mpf(KAPPA)
    mu = _mpf(BETA) * mp.pi ** 2 / 3
    return 1 + kappa - kappa / (1 + mu * s2 / kappa)


def ex_pbe(n, sigma):
    """PBE exchange energy per volume of an unpolarised density n with contracted gradient sigma."""
    kf = mp.cbrt(3 * mp.pi ** 2 * n)
    return ex_lda(n) * pbe_fx(sigma / (4 * kf ** 2 * n ** 2))


def pbe_h(n, spin, sigma, ec):
    """PBE gradient correction H per particle on the uniform-gas correlation ec."""
    beta, gamma = _mpf(BETA), _gamma()
    phi = 1 if spin is None else (_opz_pow(spin[1], mp.mpf(2) / 3) + _opz_pow(spin[2], mp.mpf(2) / 3)) / 2
    kf = mp.cbrt(3 * mp.pi ** 2 * n)
    ks2 = 4 * kf / mp.pi
    t2 = sigma / (4 * phi ** 2 * ks2 * n ** 2)
    A = beta / gamma / (mp.exp(-ec / (gamma * phi ** 3)) - 1)
    At2 = A * t2
    return gamma * phi ** 3 * mp.log(1 + beta / gamma * t2 * (1 + At2) / (1 + At2 + At2 ** 2))


def energy(functional, rho, sigma):
    """Energy per volume of one functional, before any flooring of the inputs.  rho: (n,) or (up, dn);
    sigma: () or (s,) or (uu, ud, dd)."""
    polarised = len(rho) == 2
    n = rho[0] + rho[1] if polarised else rho[0]
    spin = ((rho[0] - rho[1]) / n, 2 * rho[0] / n, 2 * rho[1] / n) if polarised else None
    rs = mp.cbrt(3 / (4 * mp.pi * n))
    if functional in ("lda_x", "gga_x_pbe"):
        def channel(r, s):
            return ex_lda(r) if functional == "lda_x" else ex_pbe(r, s)
        if not polarised:
            return channel(n, sigma[0] if sigma else 0)
        total = mp.mpf(0)
        for r, s in ((rho[0], sigma[0] if sigma else 0), (rho[1], sigma[2] if sigma else 0)):
            if r > DENS_THRESHOLD_SPIN:
                total += channel(2 * r, 4 * s) / 2
        return total
    if functional == "lda_c_vwn":
        return n * eps_c_lda(rs, spin, "vwn")
    if functional == "lda_c_pw":
        return n * eps_c_lda(rs, spin, "pw")
    if functional == "gga_c_pbe":
        st = sigma[0] if not polarised else sigma[0] + 2 * sigma[1] + sigma[2]
        ec = eps_c_lda(rs, spin, "pw_mod")
        return n * (ec + pbe_h(n, spin, st, ec))
    raise NotImplementedError(functional)


def evaluate(functionals, rho, sigma=()):
    """e, vrho, vsigma of a sum of functionals at one point, as the mpf values libxc would return as zk * rho, vrho
    and vsigma.  rho: (n,) or (up, dn) floats; sigma: () for LDA, (s,) or (uu, ud, dd) for GGA."""
    with mp.workdps(DPS):
        rho = [_mpf(float(r)) for r in rho]
        sigma = [_mpf(float(s)) for s in sigma]
        nv = len(rho) + len(sigma)
        if not sum(rho) > DENS_THRESHOLD:
            return mp.mpf(0), [mp.mpf(0)] * len(rho), [mp.mpf(0)] * len(sigma)
        rho = [max(r, mp.mpf(0)) for r in rho]
        floored = (0,) if len(sigma) == 1 else (0, 2)
        for i in floored:
            if i < len(sigma):
                sigma[i] = max(sigma[i], _mpf(SIGMA_FLOOR))
        x0 = rho + sigma
        n = sum(rho)
        sigma_unit = 4 * mp.cbrt(3 * mp.pi ** 2) ** 2 * n ** (mp.mpf(8) / 3)   # sigma at reduced gradient s = 1

        def f(x):
            return sum(energy(fn, x[:len(rho)], x[len(rho):]) for fn in functionals)

        def partial(i):
            scale = n if i < len(rho) else sigma_unit
            h = mp.mpf("1e-25") * (abs(x0[i]) if x0[i] != 0 else scale)

            def g(t):
                x = list(x0)
                x[i] = t
                return f(x)
            return mp.diff(g, x0[i], h=h)
        d = [partial(i) for i in range(nv)]
        return f(x0), d[:len(rho)], d[len(rho):]
