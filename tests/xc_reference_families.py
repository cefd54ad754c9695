"""Extended-precision reference for the Teter-Pade and Perdew-Zunger LDAs and the PBEsol, revPBE and RPBE GGAs
(test infrastructure), on the thresholds and LDA pieces of tests/xc_reference.py.

Restated from the papers' closed forms, in mpmath at xc_reference.DPS digits:
  lda_xc_teter93  Goedecker, Teter, Hutter, Phys. Rev. B 54, 1703 (1996): exchange and correlation together,
                  eps_xc = -(a0 + a1 rs + a2 rs^2 + a3 rs^3) / (b1 rs + b2 rs^2 + b3 rs^3 + b4 rs^4), every coefficient
                  c + f(zeta) dc with f the PW92 / VWN spin interpolation
  lda_c_pz        Perdew, Zunger, Phys. Rev. B 23, 5048 (1981): gamma / (1 + beta1 sqrt(rs) + beta2 rs) for rs >= 1,
                  A ln rs + B + C rs ln rs + D rs below; eps_P + f(zeta) (eps_F - eps_P)
  gga_x_pbe_sol   Perdew et al., Phys. Rev. Lett. 100, 136406 (2008): the PBE enhancement factor with mu = 10/81
  gga_c_pbe_sol   the same paper: PBE correlation on PW92-mod with beta = 0.046
  gga_x_pbe_r     Zhang, Yang, Phys. Rev. Lett. 80, 890 (1998) (revPBE): the PBE enhancement factor with kappa = 1.245
  gga_x_rpbe      Hammer, Hansen, Norskov, Phys. Rev. B 59, 7413 (1999): F_x = 1 + kappa (1 - exp(-mu s^2 / kappa))
The Teter-Pade coefficients are libxc's as recalled, not checked against libxc's sources; with them the reference's
iron LDA setup (test/iron_lda.jl) reproduces its ABINIT energies.  vrho and vsigma are central finite differences,
as in xc_reference.  The five functionals of xc_reference are delegated to it.
"""
import mpmath as mp

import xc_reference as xr

FUNCTIONALS = ("lda_xc_teter93", "lda_c_pz", "gga_x_pbe_sol", "gga_c_pbe_sol", "gga_x_pbe_r", "gga_x_rpbe")

_TETER = dict(
    a=("0.4581652932831429", "2.217058676663745", "0.7405551735357053", "0.01968227878617998"),
    da=("0.119086804055547", "0.6157402568883345", "0.1574201515892867", "0.003532336663397157"),
    b=("1.0", "4.504130959426697", "1.110667363742916", "0.02359291751427506"),
    db=("0", "0.2673612973836267", "0.2052004607777787", "0.004200005045691381"),
)
_PZ = (   # (gamma, beta1, beta2, A, B, C, D): paramagnetic, ferromagnetic
    ("-0.1423", "1.0529", "0.3334", "0.0311", "-0.048", "0.0020", "-0.0116"),
    ("-0.0843", "1.3981", "0.2611", "0.01555", "-0.0269", "0.0007", "-0.0048"),
)
BETA_PBE_SOL = "0.046"
KAPPA_REVPBE = "1.245"


def _mu_pbe():
    return mp.mpf(xr.BETA) * mp.pi ** 2 / 3


def eps_xc_teter(rs, spin):
    """Teter-Pade exchange-correlation energy per particle.  spin = None or (zeta, 1 + zeta, 1 - zeta)."""
    f = 0 if spin is None else xr._f_zeta(spin[1], spin[2])
    a = [mp.mpf(c) + f * mp.mpf(d) for c, d in zip(_TETER["a"], _TETER["da"])]
    b = [mp.mpf(c) + f * mp.mpf(d) for c, d in zip(_TETER["b"], _TETER["db"])]
    return -sum(a[i] * rs ** i for i in range(4)) / sum(b[i] * rs ** (i + 1) for i in range(4))


def _pz(rs, i):
    g, b1, b2, A, B, C, D = (mp.mpf(v) for v in _PZ[i])
    if rs >= 1:
        return g / (1 + b1 * mp.sqrt(rs) + b2 * rs)
    return A * mp.log(rs) + B + C * rs * mp.log(rs) + D * rs


def eps_c_pz(rs, spin):
    """Perdew-Zunger correlation energy per particle."""
    ep = _pz(rs, 0)
    if spin is None:
        return ep
    return ep + xr._f_zeta(spin[1], spin[2]) * (_pz(rs, 1) - ep)


def fx(functional, s2):
    """The exchange enhancement factor at s^2."""
    kappa, mu = mp.mpf(xr.KAPPA), _mu_pbe()
    if functional == "gga_x_pbe_sol":
        mu = mp.mpf(10) / 81
    elif functional == "gga_x_pbe_r":
        kappa = mp.mpf(KAPPA_REVPBE)
    elif functional == "gga_x_rpbe":
        return 1 + kappa * (1 - mp.exp(-mu * s2 / kappa))
    return 1 + kappa - kappa / (1 + mu * s2 / kappa)


def ex_gga(functional, n, sigma):
    """GGA exchange energy per volume of an unpolarised density n with contracted gradient sigma."""
    kf = mp.cbrt(3 * mp.pi ** 2 * n)
    return xr.ex_lda(n) * fx(functional, sigma / (4 * kf ** 2 * n ** 2))


def pbe_h(n, spin, sigma, ec, beta):
    """PBE gradient correction H per particle with gradient coefficient beta."""
    gamma = xr._gamma()
    phi = 1 if spin is None else (xr._opz_pow(spin[1], mp.mpf(2) / 3) + xr._opz_pow(spin[2], mp.mpf(2) / 3)) / 2
    kf = mp.cbrt(3 * mp.pi ** 2 * n)
    t2 = sigma / (4 * phi ** 2 * (4 * kf / mp.pi) * n ** 2)
    A = beta / gamma / (mp.exp(-ec / (gamma * phi ** 3)) - 1)
    At2 = A * t2
    return gamma * phi ** 3 * mp.log(1 + beta / gamma * t2 * (1 + At2) / (1 + At2 + At2 ** 2))


def energy(functional, rho, sigma):
    """Energy per volume of one functional, before any flooring of the inputs (as xc_reference.energy)."""
    if functional not in FUNCTIONALS:
        return xr.energy(functional, rho, sigma)
    polarised = len(rho) == 2
    n = rho[0] + rho[1] if polarised else rho[0]
    spin = ((rho[0] - rho[1]) / n, 2 * rho[0] / n, 2 * rho[1] / n) if polarised else None
    rs = mp.cbrt(3 / (4 * mp.pi * n))
    if functional == "lda_xc_teter93":
        return n * eps_xc_teter(rs, spin)
    if functional == "lda_c_pz":
        return n * eps_c_pz(rs, spin)
    if functional == "gga_c_pbe_sol":
        st = sigma[0] if not polarised else sigma[0] + 2 * sigma[1] + sigma[2]
        ec = xr.eps_c_lda(rs, spin, "pw_mod")
        return n * (ec + pbe_h(n, spin, st, ec, mp.mpf(BETA_PBE_SOL)))
    if not polarised:
        return ex_gga(functional, n, sigma[0])
    total = mp.mpf(0)
    for r, s in ((rho[0], sigma[0]), (rho[1], sigma[2])):
        if r > xr.DENS_THRESHOLD_SPIN:
            total += ex_gga(functional, 2 * r, 4 * s) / 2
    return total


def evaluate(functionals, rho, sigma=()):
    """e, vrho, vsigma of a sum of functionals at one point, with the input flooring of xc_reference.evaluate."""
    with mp.workdps(xr.DPS):
        rho = [mp.mpf(float(r)) for r in rho]
        sigma = [mp.mpf(float(s)) for s in sigma]
        if not sum(rho) > xr.DENS_THRESHOLD:
            return mp.mpf(0), [mp.mpf(0)] * len(rho), [mp.mpf(0)] * len(sigma)
        rho = [max(r, mp.mpf(0)) for r in rho]
        for i in ((0,) if len(sigma) == 1 else (0, 2)):
            if i < len(sigma):
                sigma[i] = max(sigma[i], mp.mpf(xr.SIGMA_FLOOR))
        x0 = rho + sigma
        n = sum(rho)
        sigma_unit = 4 * mp.cbrt(3 * mp.pi ** 2) ** 2 * n ** (mp.mpf(8) / 3)

        def f(x):
            return sum(energy(fn, x[:len(rho)], x[len(rho):]) for fn in functionals)

        def partial(i):
            h = mp.mpf("1e-25") * (abs(x0[i]) if x0[i] != 0 else (n if i < len(rho) else sigma_unit))

            def g(t):
                x = list(x0)
                x[i] = t
                return f(x)
            return mp.diff(g, x0[i], h=h)
        d = [partial(i) for i in range(len(x0))]
        return f(x0), d[:len(rho)], d[len(rho):]
