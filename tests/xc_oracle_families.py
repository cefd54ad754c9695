"""The Teter-Pade and Perdew-Zunger LDAs and the PBEsol, revPBE and RPBE GGAs for the CPU oracle (test infrastructure).

`evaluate` extends oracle.xc.evaluate by these six functionals, on the oracle's NumPy dual numbers and with its edge
semantics, and leaves the oracle's own functionals to it.  `install(monkeypatch)` puts it in place of
oracle.xc.evaluate, which every oracle XC evaluation (oracle.terms.xc_potential, and through it oracle.nlcc and the
SCF) looks up at call time.  The closed forms and constants are those of the kernel (csrc/xc_core.cuh) and of
tests/xc_reference_families.py.
"""
import math
import numpy as np

import oracle.xc as ox

NEW = ("lda_xc_teter93", "lda_c_pz", "gga_x_pbe_sol", "gga_c_pbe_sol", "gga_x_pbe_r", "gga_x_rpbe")
_BASE = ox.evaluate

_TETER_A = (0.4581652932831429, 2.217058676663745, 0.7405551735357053, 0.01968227878617998)
_TETER_DA = (0.119086804055547, 0.6157402568883345, 0.1574201515892867, 0.003532336663397157)
_TETER_B = (1.0, 4.504130959426697, 1.110667363742916, 0.02359291751427506)
_TETER_DB = (0.0, 0.2673612973836267, 0.2052004607777787, 0.004200005045691381)
_PZ = ((-0.1423, 1.0529, 0.3334, 0.0311, -0.048, 0.0020, -0.0116),
       (-0.0843, 1.3981, 0.2611, 0.01555, -0.0269, 0.0007, -0.0048))


def _exc_teter(rs, spin):
    f = 0.0 if spin is None else ox._fzeta(spin)
    a = [c + d * f for c, d in zip(_TETER_A, _TETER_DA)]
    b = [c + d * f for c, d in zip(_TETER_B, _TETER_DB)]
    num = a[0] + rs * (a[1] + rs * (a[2] + rs * a[3]))
    den = rs * (b[0] + rs * (b[1] + rs * (b[2] + rs * b[3])))
    return -1.0 * num / den


def _pz_piece(rs, p):
    g, b1, b2, A, B, C, D = p
    hi = rs.v >= 1.0                 # each branch is evaluated at a placeholder where the other one holds
    lo_rs = ox.Dual(np.where(hi, 0.5, rs.v), rs.d)
    low = A * ox.dlog(lo_rs) + B + C * lo_rs * ox.dlog(lo_rs) + D * lo_rs
    hi_rs = ox.Dual(np.where(hi, rs.v, 1.0), rs.d)
    high = g / (1 + b1 * ox.dsqrt(hi_rs) + b2 * hi_rs)
    return ox.Dual(np.where(hi, high.v, low.v), np.where(hi[None, :], high.d, low.d))


def _ec_pz(rs, spin):
    ep = _pz_piece(rs, _PZ[0])
    if spin is None:
        return ep
    return ep + ox._fzeta(spin) * (_pz_piece(rs, _PZ[1]) - ep)


def _ex_gga(functional, rho, sigma):
    kappa, mu = ox._KAPPA, ox._MU
    if functional == "gga_x_pbe_sol":
        mu = 10 / 81
    elif functional == "gga_x_pbe_r":
        kappa = 1.245
    kF = ox.dcbrt(3 * math.pi ** 2 * rho)
    s2 = sigma / (4 * kF * kF * rho * rho)
    if functional == "gga_x_rpbe":
        Fx = 1 - kappa * ox.dexpm1((-mu / kappa) * s2)
    else:
        Fx = 1 + kappa - kappa / (1 + mu * s2 / kappa)
    return ox._ex_unif_unpol(rho) * Fx


def _ec_pbe_sol(rho, rs, spin, sigma_tot):
    beta, gamma = 0.046, ox._GAMMA
    ec = ox._ec_pw(rs, spin, ox._PWMOD)
    if spin is None:
        phi, phi3 = 1.0, 1.0
    else:
        phi = (ox._opz_pow(spin[1], 2 / 3) + ox._opz_pow(spin[2], 2 / 3)) / 2
        phi3 = phi * phi * phi
    kF = ox.dcbrt(3 * math.pi ** 2 * rho)
    t2 = sigma_tot / (4 * (phi * phi) * (4 * kF / math.pi) * rho * rho)
    A = (beta / gamma) / ox.dexpm1(-ec / (gamma * phi3))
    At2 = A * t2
    return ec + gamma * phi3 * ox.dlog1p((beta / gamma) * t2 * (1 + At2) / (1 + At2 + At2 * At2))


def _evaluate_new(functionals, rho, sigma, is_gga):
    """The part of evaluate for the six functionals of NEW (the setup of oracle.xc.evaluate).  is_gga: whether the
    whole set, not only this part, takes sigma."""
    n_spin, N = rho.shape
    nvar = n_spin + (sigma.shape[0] if is_gga else 0)
    mask = rho.sum(axis=0) > ox.DENS_THRESHOLD
    safe = np.where(mask, rho, 1.0 / n_spin)

    def var(i, val):
        d = np.zeros((nvar, N))
        d[i] = 1.0
        return ox.Dual(val.copy(), d)

    r = [var(s, np.maximum(safe[s], 0.0)) for s in range(n_spin)]
    sg = None
    if is_gga:
        ssafe = np.where(mask, sigma, 0.0)
        floored = [0] if sigma.shape[0] == 1 else [0, 2]
        ssafe[floored] = np.maximum(ssafe[floored], ox.SIGMA_FLOOR)
        sg = [var(n_spin + i, ssafe[i]) for i in range(sigma.shape[0])]
    n = r[0] if n_spin == 1 else r[0] + r[1]
    spin = None if n_spin == 1 else ((r[0] - r[1]) / n, 2 * r[0] / n, 2 * r[1] / n)
    rs = ox._RS_FAC / ox.dcbrt(n)

    def screened(s, piece):
        live = r[s].v > ox.DENS_THRESHOLD_SPIN
        x = piece(ox.Dual(np.where(live, r[s].v, 1.0), r[s].d))
        return ox.Dual(np.where(live, x.v, 0.0), np.where(live[None, :], x.d, 0.0))
    e = ox.Dual(np.zeros(N), np.zeros((nvar, N)))
    for f in functionals:
        if f == "lda_xc_teter93":
            e = e + n * _exc_teter(rs, spin)
        elif f == "lda_c_pz":
            e = e + n * _ec_pz(rs, spin)
        elif f == "gga_c_pbe_sol":
            stot = sg[0] if n_spin == 1 else sg[0] + 2 * sg[1] + sg[2]
            e = e + n * _ec_pbe_sol(n, rs, spin, stot)
        elif n_spin == 1:
            e = e + _ex_gga(f, n, sg[0])
        else:
            for s, isg in ((0, 0), (1, 2)):
                e = e + screened(s, lambda rr: 0.5 * _ex_gga(f, 2 * rr, 4 * sg[isg]))
    return np.where(mask, e.v, 0.0), np.where(mask[None, :], e.d, 0.0)


def evaluate(functionals, rho, sigma=None):
    """oracle.xc.evaluate over the oracle's functionals and those of NEW: the same arguments and results."""
    new = [f for f in functionals if f in NEW]
    old = [f for f in functionals if f not in NEW]
    if not new:
        return _BASE(functionals, rho, sigma)
    n_spin = rho.shape[0]
    is_gga = any(f.startswith("gga") for f in functionals)
    if is_gga:
        assert sigma is not None
    ev, dv = _evaluate_new(new, rho, sigma, is_gga)
    vsig = dv[n_spin:] if is_gga else None
    vrho = dv[:n_spin]
    if old:
        base = _BASE(old, rho, sigma)
        ev, vrho = ev + base["e"], vrho + base["Vrho"]
        if is_gga and base["Vsigma"] is not None:
            vsig = vsig + base["Vsigma"]
    return dict(e=ev, Vrho=vrho, Vsigma=vsig)


def install(monkeypatch):
    """Let the oracle evaluate the six functionals of NEW for the rest of a test."""
    monkeypatch.setattr(ox, "evaluate", evaluate)
