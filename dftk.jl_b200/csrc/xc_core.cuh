// Pointwise exchange-correlation functionals and the density symmetrisation gather (device side of the SCF
// plumbing next to the hot path, SURVEY §8f rank 1; K16 of SURVEY §2.5).
//
// XC: the reference evaluates libxc through Libxc.jl (src/DispatchFunctional.jl:55-56,108-128; call site
// src/terms/xc.jl:104-113).  libxc is third-party code that is not under the DFTK.jl tree; the closed forms are
// restated here (Dirac exchange, VWN5, PW92 / PW92-mod, Teter-Pade, Perdew-Zunger, and the PBE, PBEsol, revPBE and
// RPBE GGAs) with libxc's constants.  Energies per volume `e` and the derivatives vrho / vsigma come from ONE
// expression evaluated on forward-mode dual numbers, so they are mutually consistent by construction.
//
// Bodies are __host__ __device__ (host emulation in tests/hostemu).
#pragma once
#include <math.h>
#include "fft_core.cuh"

namespace dftk {

template <int NV>
struct Dual {
  double v;
  double d[NV];
};
template <int NV>
HD Dual<NV> dconst(double c) {
  Dual<NV> r;
  r.v = c;
#pragma unroll
  for (int i = 0; i < NV; ++i) r.d[i] = 0.0;
  return r;
}
template <int NV>
HD Dual<NV> dvar(double x, int idx) {
  Dual<NV> r = dconst<NV>(x);
  r.d[idx] = 1.0;
  return r;
}
#define DUAL_BIN(op, VEXPR, DEXPR)                                      \
  template <int NV>                                                     \
  HD Dual<NV> operator op(const Dual<NV>& a, const Dual<NV>& b) {       \
    Dual<NV> r;                                                         \
    r.v = VEXPR;                                                        \
    _Pragma("unroll") for (int i = 0; i < NV; ++i) r.d[i] = DEXPR;      \
    return r;                                                           \
  }
DUAL_BIN(+, a.v + b.v, a.d[i] + b.d[i])
DUAL_BIN(-, a.v - b.v, a.d[i] - b.d[i])
DUAL_BIN(*, a.v * b.v, a.d[i] * b.v + b.d[i] * a.v)
DUAL_BIN(/, a.v / b.v, (a.d[i] - b.d[i] * (a.v / b.v)) / b.v)
#undef DUAL_BIN
template <int NV> HD Dual<NV> operator+(const Dual<NV>& a, double c) { Dual<NV> r = a; r.v += c; return r; }
template <int NV> HD Dual<NV> operator+(double c, const Dual<NV>& a) { return a + c; }
template <int NV> HD Dual<NV> operator-(const Dual<NV>& a, double c) { return a + (-c); }
template <int NV>
HD Dual<NV> operator-(const Dual<NV>& a) {
  Dual<NV> r;
  r.v = -a.v;
#pragma unroll
  for (int i = 0; i < NV; ++i) r.d[i] = -a.d[i];
  return r;
}
template <int NV> HD Dual<NV> operator-(double c, const Dual<NV>& a) { return (-a) + c; }
template <int NV>
HD Dual<NV> operator*(const Dual<NV>& a, double c) {
  Dual<NV> r;
  r.v = a.v * c;
#pragma unroll
  for (int i = 0; i < NV; ++i) r.d[i] = a.d[i] * c;
  return r;
}
template <int NV> HD Dual<NV> operator*(double c, const Dual<NV>& a) { return a * c; }
template <int NV> HD Dual<NV> operator/(const Dual<NV>& a, double c) { return a * (1.0 / c); }
template <int NV> HD Dual<NV> operator/(double c, const Dual<NV>& a) { return dconst<NV>(c) / a; }
template <int NV>
HD Dual<NV> dchain(const Dual<NV>& a, double fv, double g) {   // f(a) with f(a.v) = fv, f'(a.v) = g
  Dual<NV> r;
  r.v = fv;
#pragma unroll
  for (int i = 0; i < NV; ++i) r.d[i] = a.d[i] * g;
  return r;
}
template <int NV> HD Dual<NV> dlog(const Dual<NV>& a) { return dchain(a, log(a.v), 1.0 / a.v); }
template <int NV> HD Dual<NV> dexp(const Dual<NV>& a) { double e = exp(a.v); return dchain(a, e, e); }
template <int NV> HD Dual<NV> dlog1p(const Dual<NV>& a) { return dchain(a, log1p(a.v), 1.0 / (1.0 + a.v)); }
template <int NV> HD Dual<NV> dexpm1(const Dual<NV>& a) { return dchain(a, expm1(a.v), exp(a.v)); }
template <int NV> HD Dual<NV> dsqrt(const Dual<NV>& a) { double q = sqrt(a.v); return dchain(a, q, 0.5 / q); }
template <int NV> HD Dual<NV> datan(const Dual<NV>& a) { return dchain(a, atan(a.v), 1.0 / (1.0 + a.v * a.v)); }
template <int NV> HD Dual<NV> dcbrt(const Dual<NV>& a) { double c = cbrt(a.v); return dchain(a, c, c / (3.0 * a.v)); }
template <int NV> HD Dual<NV> dpow(const Dual<NV>& a, double p) { return dchain(a, pow(a.v, p), p * pow(a.v, p - 1.0)); }

#define XC_LDA_X 1
#define XC_LDA_C_VWN 2
#define XC_LDA_C_PW 4
#define XC_GGA_X_PBE 8
#define XC_GGA_C_PBE 16
#define XC_LDA_XC_TETER93 32
#define XC_LDA_C_PZ 64
#define XC_GGA_X_PBE_SOL 128
#define XC_GGA_C_PBE_SOL 256
#define XC_GGA_X_PBE_R 512
#define XC_GGA_X_RPBE 1024
// the functionals that need the contracted gradient sigma, and every bit the kernel knows
#define XC_GGA_BITS (XC_GGA_X_PBE | XC_GGA_C_PBE | XC_GGA_X_PBE_SOL | XC_GGA_C_PBE_SOL | XC_GGA_X_PBE_R | XC_GGA_X_RPBE)
#define XC_VALID_BITS (XC_LDA_X | XC_LDA_C_VWN | XC_LDA_C_PW | XC_LDA_XC_TETER93 | XC_LDA_C_PZ | XC_GGA_BITS)
// Edge semantics of libxc (restated from its documented behaviour; the values are not checked against libxc's
// sources in this tree):
//   XC_DENS_THRESHOLD       a point whose total density is at or below it gives zero energy and potentials;
//   XC_DENS_THRESHOLD_SPIN  a spin channel at or below it contributes nothing to spin-resolved exchange (value and
//                           derivatives), so a fully polarised point has finite minority potentials;
//   XC_ZETA_THRESHOLD       (1 +- zeta)^p at or below it is frozen at the threshold with zero derivative (DBL_EPSILON);
//   XC_SIGMA_FLOOR          sigma_uu, sigma_dd (and the unpolarised sigma) are raised to it before evaluation, the
//                           derivatives taken at the raised value: (threshold^(4/3))^2 of the 1e-15 density threshold.
// A negative spin density (round-off, or the extrapolation of a density mixer next to an empty channel) is raised to
// zero before zeta is formed, the derivatives taken there, so |zeta| <= 1 always: left alone, zeta^4 and (1 + zeta)^p
// would be extrapolated without bound (an H-atom LDA SCF diverged this way, to eigenvalues of -2e8 Ha).  libxc is
// recalled to raise each spin density to the functional's density threshold instead (1e-12 for gga_c_pbe), which at
// rho_dn = 0 leaves phi'(zeta) evaluated at 1 - zeta = 2 threshold / n, tens of Ha in vrho_dn at n = 0.1; that floor is
// not adopted here and, like the values above, is not checked against libxc's sources.
#define XC_DENS_THRESHOLD 1e-15
#define XC_DENS_THRESHOLD_SPIN 1e-15
#define XC_ZETA_THRESHOLD 2.220446049250313e-16
#define XC_SIGMA_FLOOR 1e-40

#define XC_PI 3.14159265358979323846
// (1 + zeta)^p given opz = 1 + zeta, frozen below the zeta threshold
template <class T> HD T xc_opz_pow(const T& opz, double p) {
  if (opz.v <= XC_ZETA_THRESHOLD) return dchain(opz, pow(XC_ZETA_THRESHOLD, p), 0.0);
  return dpow(opz, p);
}
// Spin variables of a polarised point: zeta and 1 +- zeta, the latter formed as 2 rho_s / n so that they keep
// their relative precision as zeta -> +-1.
template <class T> struct XcSpin { T z, opz, omz; };
template <class T> HD T xc_fzeta(const XcSpin<T>& sp) {
  return (xc_opz_pow(sp.opz, 4.0 / 3.0) + xc_opz_pow(sp.omz, 4.0 / 3.0) - 2.0) / (2.5198420997897464 - 2.0);   // 2^(4/3) - 2
}
template <class T> HD T xc_ex_unif(const T& n) { return (-0.75 * 0.98474502184269641) * n * dcbrt(n); }   // (3/pi)^(1/3)

template <class T>
HD T xc_vwn_piece(const T& x, double A, double b, double c, double x0) {
  const double Q = sqrt(4.0 * c - b * b);
  T X = x * x + b * x + c;
  const double X0 = x0 * x0 + b * x0 + c;
  T at = datan(Q / (2.0 * x + b));
  return A * (dlog(x * x / X) + (2.0 * b / Q) * at -
              (b * x0 / X0) * (dlog((x - x0) * (x - x0) / X) + (2.0 * (b + 2.0 * x0) / Q) * at));
}
template <class T>
HD T xc_ec_vwn(const T& rs, const XcSpin<T>* sp) {
  T x = dsqrt(rs);
  T p0 = xc_vwn_piece(x, 0.0310907, 3.72744, 12.9352, -0.10498);
  if (!sp) return p0;
  T p1 = xc_vwn_piece(x, 0.01554535, 7.06042, 18.0578, -0.32500);
  T p2 = xc_vwn_piece(x, -1.0 / (6.0 * XC_PI * XC_PI), 1.13107, 13.0045, -0.0047584);
  T fz = xc_fzeta(*sp);
  T z2 = sp->z * sp->z;
  T z4 = z2 * z2;
  const double fpp0 = 4.0 / (9.0 * (1.2599210498948732 - 1.0));   // 4 / (9 (2^(1/3) - 1))
  return p0 + p2 * fz * (1.0 - z4) / fpp0 + (p1 - p0) * fz * z4;
}
template <class T>
HD T xc_pw_G(const T& rs, double a, double a1, double b1, double b2, double b3, double b4) {
  T s = dsqrt(rs);
  T den = (2.0 * a) * (b1 * s + b2 * rs + b3 * rs * s + b4 * rs * rs);
  return (-2.0 * a) * (1.0 + a1 * rs) * dlog1p(1.0 / den);   // log1p: 1 / den -> 0 at large rs
}
template <class T>
HD T xc_ec_pw(const T& rs, const XcSpin<T>* sp, bool mod) {
  const double a0 = mod ? 0.0310906908696548950 : 0.0310907, a1 = mod ? 0.01554534543482744750 : 0.01554535,
               a2 = mod ? 0.0168868639404617 : 0.0168869, fz20 = mod ? 1.709920934161365617563962776245 : 1.709921;
  T g0 = xc_pw_G(rs, a0, 0.21370, 7.5957, 3.5876, 1.6382, 0.49294);
  if (!sp) return g0;
  T g1 = xc_pw_G(rs, a1, 0.20548, 14.1189, 6.1977, 3.3662, 0.62517);
  T mac = xc_pw_G(rs, a2, 0.11125, 10.357, 3.6231, 0.88026, 0.49671);
  T fz = xc_fzeta(*sp);
  T z2 = sp->z * sp->z;
  T z4 = z2 * z2;
  return g0 - mac * fz * (1.0 - z4) / fz20 + (g1 - g0) * fz * z4;
}
// Goedecker, Teter, Hutter, Phys. Rev. B 54, 1703 (1996): the Pade fit of exchange and correlation together,
// e_xc per electron = -(a0 + a1 rs + a2 rs^2 + a3 rs^3) / (b1 rs + b2 rs^2 + b3 rs^3 + b4 rs^4), every coefficient
// c + f(zeta) dc.  The constants are libxc's lda_xc_teter93 as recalled, not checked against libxc's sources; with
// them the reference's iron LDA setup (test/iron_lda.jl) reproduces its ABINIT energy and eigenvalues.
template <class T>
HD T xc_exc_teter(const T& rs, const XcSpin<T>* sp) {
  const double a[4] = {0.4581652932831429, 2.217058676663745, 0.7405551735357053, 0.01968227878617998};
  const double da[4] = {0.119086804055547, 0.6157402568883345, 0.1574201515892867, 0.003532336663397157};
  const double b[4] = {1.0, 4.504130959426697, 1.110667363742916, 0.02359291751427506};
  const double db[4] = {0.0, 0.2673612973836267, 0.2052004607777787, 0.004200005045691381};
  if (!sp) return -(a[0] + rs * (a[1] + rs * (a[2] + rs * a[3]))) / (rs * (b[0] + rs * (b[1] + rs * (b[2] + rs * b[3]))));
  T fz = xc_fzeta(*sp);
  T num = (a[0] + da[0] * fz) + rs * ((a[1] + da[1] * fz) + rs * ((a[2] + da[2] * fz) + rs * (a[3] + da[3] * fz)));
  T den = rs * ((b[0] + db[0] * fz) + rs * ((b[1] + db[1] * fz) + rs * ((b[2] + db[2] * fz) + rs * (b[3] + db[3] * fz))));
  return -num / den;
}
// Perdew, Zunger, Phys. Rev. B 23, 5048 (1981): gamma / (1 + beta1 sqrt(rs) + beta2 rs) for rs >= 1 (libxc's
// branch point), A ln rs + B + C rs ln rs + D rs below, in the paramagnetic and ferromagnetic limits, interpolated
// with f(zeta).  The paper's constants.
template <class T>
HD T xc_pz_piece(const T& rs, double gamma, double beta1, double beta2, double A, double B, double C, double D) {
  if (rs.v >= 1.0) return gamma / (1.0 + beta1 * dsqrt(rs) + beta2 * rs);
  T lr = dlog(rs);
  return A * lr + B + C * rs * lr + D * rs;
}
template <class T>
HD T xc_ec_pz(const T& rs, const XcSpin<T>* sp) {
  T ep = xc_pz_piece(rs, -0.1423, 1.0529, 0.3334, 0.0311, -0.048, 0.0020, -0.0116);
  if (!sp) return ep;
  T ef = xc_pz_piece(rs, -0.0843, 1.3981, 0.2611, 0.01555, -0.0269, 0.0007, -0.0048);
  return ep + xc_fzeta(*sp) * (ef - ep);
}
#define XC_KAPPA 0.8040
#define XC_BETA 0.06672455060314922
#define XC_MU_PBE (XC_BETA * (XC_PI * XC_PI / 3.0))
// The PBE enhancement factor 1 + kappa - kappa / (1 + mu s^2 / kappa): PBE (kappa 0.804, mu_PBE), PBEsol (Perdew et
// al., Phys. Rev. Lett. 100, 136406 (2008): mu = 10/81) and revPBE (Zhang, Yang, Phys. Rev. Lett. 80, 890 (1998):
// kappa = 1.245).  The call sites pass literals, so each folds to its constants.
template <class T>
HD T xc_ex_pbe(const T& n, const T& sigma, double kappa, double mu) {
  T kF = dcbrt((3.0 * XC_PI * XC_PI) * n);
  T s2 = sigma / (4.0 * kF * kF * n * n);
  return xc_ex_unif(n) * ((1.0 + kappa) - kappa / (1.0 + (mu / kappa) * s2));
}
// RPBE (Hammer, Hansen, Norskov, Phys. Rev. B 59, 7413 (1999)): F_x = 1 + kappa (1 - exp(-mu s^2 / kappa)).
template <class T>
HD T xc_ex_rpbe(const T& n, const T& sigma) {
  T kF = dcbrt((3.0 * XC_PI * XC_PI) * n);
  T s2 = sigma / (4.0 * kF * kF * n * n);
  return xc_ex_unif(n) * (1.0 - XC_KAPPA * dexpm1((-XC_MU_PBE / XC_KAPPA) * s2));
}
// The GGA exchange of mask bit BIT, for an unpolarised density n with contracted gradient sigma.
template <int BIT, class T>
HD T xc_ex_gga(const T& n, const T& sigma) {
  if (BIT == XC_GGA_X_PBE) return xc_ex_pbe(n, sigma, XC_KAPPA, XC_MU_PBE);
  if (BIT == XC_GGA_X_PBE_SOL) return xc_ex_pbe(n, sigma, XC_KAPPA, 10.0 / 81.0);
  if (BIT == XC_GGA_X_PBE_R) return xc_ex_pbe(n, sigma, 1.245, XC_MU_PBE);
  return xc_ex_rpbe(n, sigma);
}
// acc += that exchange at a point, spin-resolved as (E[2 rho_up, 4 sigma_uu] + E[2 rho_dn, 4 sigma_dd]) / 2 with a
// channel at or below XC_DENS_THRESHOLD_SPIN left out.  r: NSPIN densities, sg: NSIG contracted gradients.
template <int BIT, int NSPIN, int NSIG, class T>
HD void xc_add_ex_gga(T& acc, const T& n, const T* r, const T* sg) {
  if (NSPIN == 1) {
    acc = acc + xc_ex_gga<BIT>(n, sg[0]);
    return;
  }
  if (r[0].v > XC_DENS_THRESHOLD_SPIN) acc = acc + 0.5 * xc_ex_gga<BIT>(2.0 * r[0], 4.0 * sg[0]);
  if (r[NSPIN - 1].v > XC_DENS_THRESHOLD_SPIN) acc = acc + 0.5 * xc_ex_gga<BIT>(2.0 * r[NSPIN - 1], 4.0 * sg[NSIG - 1]);
}
// PBE correlation on PW92-mod with gradient coefficient beta: beta_PBE, or 0.046 for PBEsol.
template <class T>
HD T xc_ec_pbe(const T& n, const T& rs, const XcSpin<T>* sp, const T& sigma, double beta) {
  const double gamma = (1.0 - 0.69314718055994531) / (XC_PI * XC_PI);
  T ec = xc_ec_pw(rs, sp, true);
  T phi2 = ec * 0.0 + 1.0, phi3 = ec * 0.0 + 1.0;
  if (sp) {
    T phi = (xc_opz_pow(sp->opz, 2.0 / 3.0) + xc_opz_pow(sp->omz, 2.0 / 3.0)) * 0.5;
    phi2 = phi * phi;
    phi3 = phi2 * phi;
  }
  T kF = dcbrt((3.0 * XC_PI * XC_PI) * n);
  T t2 = sigma / (4.0 * phi2 * ((4.0 / XC_PI) * kF) * n * n);
  T Aa = (beta / gamma) / dexpm1(-ec / (gamma * phi3));
  T At2 = Aa * t2;
  return ec + gamma * phi3 * dlog1p((beta / gamma) * t2 * (1.0 + At2) / (1.0 + At2 + At2 * At2));
}

// One grid point.  rho: n_spin values; sigma: 1 (unpolarised) or 3 (uu, ud, dd) values, ignored for LDA.
// NV = n_spin (LDA) or n_spin + n_sigma (GGA).  Outputs: e, vrho[n_spin], vsigma[n_sigma].
template <int NSPIN, bool GGA>
HD void xc_point(int mask, const double* rho, const double* sigma, double* e, double* vrho, double* vsigma) {
  constexpr int NSIG = GGA ? (NSPIN == 1 ? 1 : 3) : 0;
  constexpr int NV = NSPIN + NSIG;
  typedef Dual<NV> T;
  double tot = 0.0;
  for (int s = 0; s < NSPIN; ++s) tot += rho[s];
  if (!(tot > XC_DENS_THRESHOLD)) {
    *e = 0.0;
    for (int s = 0; s < NSPIN; ++s) vrho[s] = 0.0;
    for (int s = 0; s < NSIG; ++s) vsigma[s] = 0.0;
    return;
  }
  T r[NSPIN];
  for (int s = 0; s < NSPIN; ++s) {
    r[s] = dvar<NV>(rho[s], s);
    if (r[s].v < 0.0) r[s].v = 0.0;   // only reachable for NSPIN == 2: the total is above the threshold
  }
  T sg[NSIG > 0 ? NSIG : 1];
  for (int s = 0; s < NSIG; ++s) {
    sg[s] = dvar<NV>(sigma[s], NSPIN + s);
    if (s != 1 && sg[s].v < XC_SIGMA_FLOOR) sg[s].v = XC_SIGMA_FLOOR;   // sigma_ud (s == 1) is not floored
  }
  T n = r[0];
  XcSpin<T> sp;
  if (NSPIN == 2) {
    n = r[0] + r[1];
    sp.z = (r[0] - r[1]) / n;
    sp.opz = 2.0 * r[0] / n;
    sp.omz = 2.0 * r[1] / n;
  }
  const XcSpin<T>* spp = NSPIN == 2 ? &sp : nullptr;
  T rs = 0.62035049089940009 / dcbrt(n);   // (3/(4 pi))^(1/3)
  T acc = dconst<NV>(0.0);
  if (mask & XC_LDA_X) {
    if (NSPIN == 1) acc = acc + xc_ex_unif(n);
    else
      for (int s = 0; s < NSPIN; ++s)
        if (r[s].v > XC_DENS_THRESHOLD_SPIN) acc = acc + 0.5 * xc_ex_unif(2.0 * r[s]);
  }
  if (mask & XC_LDA_C_VWN) acc = acc + n * xc_ec_vwn(rs, spp);
  if (mask & XC_LDA_C_PW) acc = acc + n * xc_ec_pw(rs, spp, false);
  if (mask & XC_LDA_XC_TETER93) acc = acc + n * xc_exc_teter(rs, spp);
  if (mask & XC_LDA_C_PZ) acc = acc + n * xc_ec_pz(rs, spp);
  if (GGA && (mask & XC_GGA_X_PBE)) xc_add_ex_gga<XC_GGA_X_PBE, NSPIN, NSIG>(acc, n, r, sg);
  if (GGA && (mask & XC_GGA_X_PBE_SOL)) xc_add_ex_gga<XC_GGA_X_PBE_SOL, NSPIN, NSIG>(acc, n, r, sg);
  if (GGA && (mask & XC_GGA_X_PBE_R)) xc_add_ex_gga<XC_GGA_X_PBE_R, NSPIN, NSIG>(acc, n, r, sg);
  if (GGA && (mask & XC_GGA_X_RPBE)) xc_add_ex_gga<XC_GGA_X_RPBE, NSPIN, NSIG>(acc, n, r, sg);
  if (GGA && (mask & (XC_GGA_C_PBE | XC_GGA_C_PBE_SOL))) {
    T st = sg[0];
    if (NSPIN == 2) st = sg[0] + 2.0 * sg[NSIG > 1 ? 1 : 0] + sg[NSIG > 2 ? 2 : 0];
    if (mask & XC_GGA_C_PBE) acc = acc + n * xc_ec_pbe(n, rs, spp, st, XC_BETA);
    if (mask & XC_GGA_C_PBE_SOL) acc = acc + n * xc_ec_pbe(n, rs, spp, st, 0.046);
  }
  *e = acc.v;
  for (int s = 0; s < NSPIN; ++s) vrho[s] = acc.d[s];
  for (int s = 0; s < NSIG; ++s) vsigma[s] = acc.d[NSPIN + s];
}

// rho, sigma, vrho, vsigma are stored component-major: x[component * N + i]
template <int NSPIN, bool GGA>
HD void xc_eval_range(int mask, int64_t i, int64_t N, const double* rho, const double* sigma, double* e,
                      double* vrho, double* vsigma) {
  constexpr int NSIG = GGA ? (NSPIN == 1 ? 1 : 3) : 0;
  double r[NSPIN], s[NSIG > 0 ? NSIG : 1], vr[NSPIN], vs[NSIG > 0 ? NSIG : 1], ee;
  for (int c = 0; c < NSPIN; ++c) r[c] = rho[c * N + i];
  for (int c = 0; c < NSIG; ++c) s[c] = sigma[c * N + i];
  xc_point<NSPIN, GGA>(mask, r, s, &ee, vr, vs);
  e[i] = ee;
  for (int c = 0; c < NSPIN; ++c) vrho[c * N + i] = vr[c];
  for (int c = 0; c < NSIG; ++c) vsigma[c * N + i] = vs[c];
}

// ---- accumulate_over_symmetries! (src/symmetry.jl:282-327): out[G] = (1/n_sym) sum_s e^{-2 pi i G.tau_s} in[S_s^-1 G]
HD int wrap_index(int g, int n) {   // integer frequency -> array index, or -1 if outside the FFT box
  const int start = -(n / 2), stop = (n - 1) / 2;
  if (g < start || g > stop) return -1;
  return g < 0 ? g + n : g;
}
HD int freq_of_index(int i, int n) { return i <= (n - 1) / 2 ? i : i - n; }
HD void symmetrize_point(int64_t idx, int nx, int ny, int nz, const cplx* __restrict__ in, cplx* __restrict__ out,
                         int n_sym, const int* __restrict__ invS, const double* __restrict__ tau) {
  const int ix = (int)(idx % nx), iy = (int)((idx / nx) % ny), iz = (int)(idx / ((int64_t)nx * ny));
  const int G[3] = {freq_of_index(ix, nx), freq_of_index(iy, ny), freq_of_index(iz, nz)};
  double ax = 0.0, ay = 0.0;
  for (int s = 0; s < n_sym; ++s) {
    const int* M = invS + 9 * s;
    const int g0 = M[0] * G[0] + M[1] * G[1] + M[2] * G[2];
    const int g1 = M[3] * G[0] + M[4] * G[1] + M[5] * G[2];
    const int g2 = M[6] * G[0] + M[7] * G[1] + M[8] * G[2];
    const int j0 = wrap_index(g0, nx), j1 = wrap_index(g1, ny), j2 = wrap_index(g2, nz);
    if (j0 < 0 || j1 < 0 || j2 < 0) continue;
    cplx v = in[j0 + (int64_t)nx * (j1 + (int64_t)ny * j2)];
    const double* t = tau + 3 * s;
    if (t[0] != 0.0 || t[1] != 0.0 || t[2] != 0.0) {
      const double ph = -2.0 * XC_PI * (G[0] * t[0] + G[1] * t[1] + G[2] * t[2]);
      v = cmul(v, make_double2(cos(ph), sin(ph)));
    }
    ax += v.x;
    ay += v.y;
  }
  out[idx] = make_double2(ax / n_sym, ay / n_sym);
}

}  // namespace dftk
