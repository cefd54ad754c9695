"""The XC kernel bodies (xc_core.cuh, compiled for the host from tests/hostemu/emu.cu) against the extended-precision
reference of tests/xc_reference.py over the whole density, spin and gradient domain, against identities that need no
restatement of the functionals, and at the fully polarised edge."""
import ctypes
import math
import os
import subprocess
import numpy as np
import pytest

import xc_reference as xr

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "hostemu", "libhostemu_xc.so")
MASK = {"lda_x": 1, "lda_c_vwn": 2, "lda_c_pw": 4, "gga_x_pbe": 8, "gga_c_pbe": 16}

# |kernel - reference| <= RTOL |reference| + ATOL * magnitude, where magnitude is the reference's own scale of the
# output at that point: E = n (|eps_x^LDA(n)| + |eps_c^PW(rs, 0)|) for e, E / n times (1 + (1 - |zeta|)^(-1/3)) for
# vrho -- the size of the phi'(zeta) and f'(zeta) terms it sums -- and E / (sigma_tot + sigma at s = 1) for vsigma.
# The absolute part covers outputs that are sums of such terms cancelling to near zero (e_c and vrho as t -> oo, vrho
# where the gradient terms balance the local ones), whose relative error the inputs' rounding does not bound.
RTOL = 1e-12
ATOL = 1e-12


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "hostemu", "emu.cu")
    csrc = os.path.join(HERE, "..", "dftk.jl_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("fft_core.cuh", "fft_plan.h", "fft_reg.cuh", "fft_radix_gen.cuh", "xc_core.cuh", "forces_core.cuh", "lobpcg_small.cuh", "i8emu_core.cuh", "fft_reg_fwd.cuh")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                               "-Wno-deprecated-gpu-targets", "-o", SO, src])
    return ctypes.CDLL(SO)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def run_emu(lib, funs, rho, sigma=None):
    """rho: (n_spin, N); sigma: (n_sigma, N) or None.  Returns e (N,), vrho (n_spin, N), vsigma (n_sigma, N) or None."""
    rho = np.ascontiguousarray(rho, dtype=float)
    n_spin, N = rho.shape
    gga = any(f.startswith("gga") for f in funs)
    nsig = (1 if n_spin == 1 else 3) if gga else 0
    sg = np.ascontiguousarray(sigma if gga else np.zeros((1, N)), dtype=float)
    e, vr, vs = np.zeros(N), np.zeros((n_spin, N)), np.zeros((max(nsig, 1), N))
    mask = sum(MASK[f] for f in funs)
    assert lib.emu_xc(mask, n_spin, int(gga), ctypes.c_int64(N), _p(rho), _p(sg), _p(e), _p(vr), _p(vs)) == 0
    return e, vr, (vs if gga else None)


# ------------------------------------------------------------------ the sweep
DENSITIES = [10.0 ** k for k in range(-14, 5)]                       # rs from about 0.03 to 3e4
S_VALUES = [0.0, 1e-4, 0.1, 1.0, 10.0, 1e3]


def sigma_unit(n):
    """sigma of a density n at reduced gradient s = 1."""
    return 4 * (3 * math.pi ** 2) ** (2 / 3) * n ** (8 / 3)


def spin_pairs(n):
    """(rho_up, rho_dn) at zeta in {0, +-1e-8, +-1e-3, +-0.5, +-(1 - 1e-6), +-(1 - 1e-12), +-(1 - 1e-15), +-1}; near
    |zeta| = 1 the minority channel is formed directly as n (1 - |zeta|) / 2 so the pair holds the intended zeta."""
    out = [(n / 2, n / 2)]
    for z in (1e-8, 1e-3, 0.5):
        out += [(n * (1 + z) / 2, n * (1 - z) / 2), (n * (1 - z) / 2, n * (1 + z) / 2)]
    for d in (1e-6, 1e-12, 1e-15, 0.0):
        mi = n * d / 2
        out += [(n - mi, mi), (mi, n - mi)]
    return out


def polarised_points(gga):
    rho, sigma = [], []
    for n in DENSITIES:
        for ru, rd in spin_pairs(n):
            if not gga:
                rho.append((ru, rd))
                continue
            for s in S_VALUES:
                # each channel at reduced gradient s for the density 2 rho_s its exchange sees
                suu, sdd = s * s * sigma_unit(2 * ru) / 4, s * s * sigma_unit(2 * rd) / 4
                for c in (0.0, 1.0, -1.0):
                    rho.append((ru, rd))
                    sigma.append((suu, c * math.sqrt(suu * sdd), sdd))
    # a minority channel below zero, at round-off and at the size a density mixer's extrapolation leaves next to an
    # empty channel (down to a raw total of 1e-6 against a majority of 1e-3), and no density at all
    for n, neg in ((1e-3, -1e-18), (0.1, -1e-18), (2.0, -1e-18), (1e-5, -1e-6), (0.1, -0.02), (1e-3, -9.99e-4)):
        rho.append((n, neg))
        sigma.append((0.3 * sigma_unit(n), 0.0, 0.0))
        rho.append((neg, n))
        sigma.append((0.0, 0.0, 0.3 * sigma_unit(n)))
    rho.append((0.0, 0.0))
    sigma.append((0.0, 0.0, 0.0))
    rho = np.array(rho).T.copy()
    return rho, (np.array(sigma[:rho.shape[1]]).T.copy() if gga else None)


def unpolarised_points(gga):
    rho, sigma = [], []
    for n in DENSITIES + [0.0]:
        for s in (S_VALUES if gga else [0.0]):
            rho.append((n,))
            sigma.append((s * s * sigma_unit(n),))
    return np.array(rho).T.copy(), (np.array(sigma).T.copy() if gga else None)


def magnitudes(rho, sigma):
    """Per point: the scales of e, vrho and vsigma used by the absolute part of the bound."""
    n = np.maximum(rho.sum(axis=0), 1e-300)
    rs = (3 / (4 * math.pi * n)) ** (1 / 3)
    ex = 0.75 * (3 / math.pi) ** (1 / 3) * n ** (1 / 3)
    ec = np.array([abs(float(xr.eps_c_lda(xr._mpf(r), None, "pw"))) for r in rs])
    e_mag = n * (ex + ec)
    st = 0.0 if sigma is None else (sigma.sum(axis=0) + (sigma[1] if sigma.shape[0] == 3 else 0))
    e_mag = np.where(rho.sum(axis=0) > 0, e_mag, 0.0)        # no density: the outputs must be exactly zero
    zf = 1.0
    if rho.shape[0] == 2:
        # 1 - |zeta| as the kernel forms it (a negative channel counts as empty); frozen points carry no such term
        m = 2 * np.maximum(rho, 0.0).min(axis=0) / np.maximum(np.maximum(rho, 0.0).sum(axis=0), 1e-300)
        zf = np.where(m <= xr.ZETA_THRESHOLD, 1.0, 1 + np.maximum(m, xr.ZETA_THRESHOLD) ** (-1 / 3))
    return e_mag, e_mag / n * zf, e_mag / (np.abs(st) + sigma_unit(n) + 1e-300)


_REF_CACHE = {}


def reference(funs, rho, sigma):
    key = (funs, rho.tobytes(), None if sigma is None else sigma.tobytes())
    if key not in _REF_CACHE:
        N = rho.shape[1]
        e, vr, vs = np.zeros(N), np.zeros(rho.shape), None if sigma is None else np.zeros(sigma.shape)
        for i in range(N):
            ee, r, s = xr.evaluate(funs, rho[:, i], () if sigma is None else sigma[:, i])
            e[i] = float(ee)
            vr[:, i] = [float(x) for x in r]
            if sigma is not None:
                vs[:, i] = [float(x) for x in s]
        _REF_CACHE[key] = (e, vr, vs)
    return _REF_CACHE[key]


def assert_close(got, ref, mag, what, rho, sigma):
    assert np.all(np.isfinite(got)), f"{what}: non-finite output"
    bound = RTOL * np.abs(ref) + ATOL * mag
    bad = np.argwhere(np.abs(got - ref) > bound)
    if bad.size:
        idx = tuple(bad[0])
        i = idx[-1]
        pt = f"rho={rho[:, i]}" + ("" if sigma is None else f" sigma={sigma[:, i]}")
        raise AssertionError(f"{what}{list(idx[:-1])}: {len(bad)} points out of bound, first at {pt}: "
                             f"kernel {got[idx]!r} reference {ref[idx]!r} bound {bound[idx]:.3g}")


@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("functional", xr.FUNCTIONALS)
def test_sweep_matches_reference(emu, functional, n_spin):
    """Each functional alone (no cancellation between exchange and correlation) over the log density grid, every
    zeta down to the fully polarised edge and every reduced gradient, against the mpmath reference."""
    gga = functional.startswith("gga")
    rho, sigma = (unpolarised_points if n_spin == 1 else polarised_points)(gga)
    e, vr, vs = run_emu(emu, (functional,), rho, sigma)
    re, rvr, rvs = reference((functional,), rho, sigma)
    me, mr, ms = magnitudes(rho, sigma)
    assert_close(e, re, me, "e", rho, sigma)
    assert_close(vr, rvr, mr[None, :], "vrho", rho, sigma)
    if gga:
        assert_close(vs, rvs, ms[None, :], "vsigma", rho, sigma)


@pytest.mark.parametrize("funs", [("lda_x", "lda_c_vwn"), ("lda_x", "lda_c_pw"), ("gga_x_pbe", "gga_c_pbe")])
def test_combined_functionals_are_the_sum(emu, funs):
    """The kernel's functional sets are the sums of their members, point by point."""
    gga = funs[0].startswith("gga")
    rho, sigma = polarised_points(gga)
    both = run_emu(emu, funs, rho, sigma)
    parts = [run_emu(emu, (f,), rho, sigma) for f in funs]
    for k in range(3 if gga else 2):
        total = sum(p[k] for p in parts)
        np.testing.assert_allclose(both[k], total, rtol=1e-14, atol=1e-14 * np.abs(total).max())


# ------------------------------------------------------------------ identities
def _grid(seed, N=400):
    rng = np.random.default_rng(seed)
    n = 10.0 ** rng.uniform(-8, 3, N)
    s = 10.0 ** rng.uniform(-3, 2, N)
    return rng, n, s * s * sigma_unit(n)


@pytest.mark.parametrize("functional", ["lda_x", "gga_x_pbe"])
def test_exchange_spin_scaling(emu, functional):
    """E_x[rho_up, rho_dn] = (E_x[2 rho_up] + E_x[2 rho_dn]) / 2 with each sigma scaled by 4."""
    rng, n, sig = _grid(1)
    z = rng.uniform(-1, 1, n.size)
    ru, rd = n * (1 + z) / 2, n * (1 - z) / 2
    suu, sdd = sig * (1 + z) ** 2 / 4, sig * (1 - z) ** 2 / 4
    sigma = np.array([suu, np.sqrt(suu * sdd), sdd])
    e, vr, vs = run_emu(emu, (functional,), np.array([ru, rd]), sigma)
    eu, vu, su = run_emu(emu, (functional,), (2 * ru)[None], (4 * suu)[None])
    ed, vd, sd = run_emu(emu, (functional,), (2 * rd)[None], (4 * sdd)[None])
    np.testing.assert_allclose(e, (eu + ed) / 2, rtol=1e-13)
    np.testing.assert_allclose(vr, np.array([vu[0], vd[0]]), rtol=1e-13)
    if functional == "gga_x_pbe":
        np.testing.assert_allclose(vs[[0, 2]], 2 * np.array([su[0], sd[0]]), rtol=1e-13)
        assert np.all(vs[1] == 0.0)


@pytest.mark.parametrize("functional", ["lda_x", "gga_x_pbe"])
def test_exchange_uniform_scaling(emu, functional):
    """e_x(lambda^3 n, lambda^8 sigma) = lambda^4 e_x(n, sigma)."""
    _, n, sig = _grid(2)
    for lam in (1e-2, 0.37, 5.0, 40.0):
        e0, _, _ = run_emu(emu, (functional,), n[None], sig[None])
        e1, _, _ = run_emu(emu, (functional,), (lam ** 3 * n)[None], (lam ** 8 * sig)[None])
        np.testing.assert_allclose(e1, lam ** 4 * e0, rtol=1e-13)


@pytest.mark.parametrize("n_spin", [1, 2])
def test_pbe_reduces_to_lda_at_zero_gradient(emu, n_spin):
    """At sigma = 0 PBE exchange is Dirac exchange and PBE correlation is PW92 with the 'mod' constants (the
    reference's PW92-mod, as the kernel carries only the original-constant PW92 as an LDA)."""
    rng, n, _ = _grid(3, 200)
    z = rng.uniform(-0.99, 0.99, n.size) if n_spin == 2 else np.zeros(n.size)
    rho = np.array([n * (1 + z) / 2, n * (1 - z) / 2]) if n_spin == 2 else n[None]
    sigma = np.zeros((3 if n_spin == 2 else 1, n.size))
    ex, vx, _ = run_emu(emu, ("gga_x_pbe",), rho, sigma)
    lx, lvx, _ = run_emu(emu, ("lda_x",), rho)
    np.testing.assert_allclose(ex, lx, rtol=1e-13)
    np.testing.assert_allclose(vx, lvx, rtol=1e-13)
    ec, _, _ = run_emu(emu, ("gga_c_pbe",), rho, sigma)
    with xr.mp.workdps(30):
        ref = []
        for i in range(n.size):
            nn = xr._mpf(float(rho[:, i].sum()))
            spin = None if n_spin == 1 else ((rho[0, i] - rho[1, i]) / nn, 2 * rho[0, i] / nn, 2 * rho[1, i] / nn)
            ref.append(float(nn * xr.eps_c_lda(xr.mp.cbrt(3 / (4 * xr.mp.pi * nn)), spin, "pw_mod")))
    np.testing.assert_allclose(ec, ref, rtol=1e-12)


@pytest.mark.parametrize("zeta", [0.0, 0.6, -1.0])
def test_pbe_correlation_vanishes_at_large_gradient(emu, zeta):
    """e_c -> 0 as t -> oo (the gradient correction cancels the uniform-gas correlation) and e_c <= 0 throughout."""
    n = np.full(9, 0.05)
    t2 = 10.0 ** np.arange(-2, 16, 2)
    phi = ((1 + zeta) ** (2 / 3) + (1 - zeta) ** (2 / 3)) / 2
    sig = t2 * 4 * phi ** 2 * (4 * (3 * math.pi ** 2 * n) ** (1 / 3) / math.pi) * n ** 2
    rho = np.array([n * (1 + zeta) / 2, n * (1 - zeta) / 2])
    z0 = np.zeros_like(n)
    e, _, _ = run_emu(emu, ("gga_c_pbe",), rho, np.array([sig, z0, z0]))
    e_lda, _, _ = run_emu(emu, ("gga_c_pbe",), rho, np.zeros((3, n.size)))
    assert np.all(e <= 0.0)
    assert np.all(np.diff(e) >= 0.0)                         # monotone towards zero
    assert abs(e[-1]) < 1e-6 * abs(e_lda[0])


def test_pbe_bounds(emu):
    """The PBE exchange enhancement stays within [1, 1 + kappa] and PBE correlation is never positive."""
    rng, n, _ = _grid(4, 2000)
    s = 10.0 ** rng.uniform(-4, 4, n.size)
    sig = s * s * sigma_unit(n)
    ex, _, _ = run_emu(emu, ("gga_x_pbe",), n[None], sig[None])
    lx, _, _ = run_emu(emu, ("lda_x",), n[None])
    fx = ex / lx
    assert np.all(fx >= 1.0 - 1e-15) and np.all(fx <= 1.804 * (1 + 1e-15))
    z = rng.uniform(-1, 1, n.size)
    rho = np.array([n * (1 + z) / 2, n * (1 - z) / 2])
    sg = np.array([sig * (1 + z) ** 2 / 4, sig * (1 - z ** 2) / 4, sig * (1 - z) ** 2 / 4])
    ec, _, _ = run_emu(emu, ("gga_c_pbe",), rho, sg)
    ec1, _, _ = run_emu(emu, ("gga_c_pbe",), n[None], sig[None])
    assert np.all(ec <= 0.0) and np.all(ec1 <= 0.0)


@pytest.mark.parametrize("funs", [("lda_x", "lda_c_vwn"), ("lda_x", "lda_c_pw"), ("gga_x_pbe", "gga_c_pbe")])
def test_spin_paths_agree_at_zeta_zero(emu, funs):
    """n_spin = 2 at rho_up = rho_dn = n / 2 reproduces n_spin = 1: e and vrho agree, and vsigma through the chain
    rule of sigma = sigma_uu + 2 sigma_ud + sigma_dd with grad rho_up = grad rho_dn = grad n / 2, i.e. every sigma_st
    = sigma / 4: vsigma_uu + vsigma_ud + vsigma_dd = 4 vsigma.  Correlation depends on sigma alone, so for it the
    chain rule holds component by component: (vsigma_uu, vsigma_ud, vsigma_dd) = (1, 2, 1) vsigma."""
    gga = funs[0].startswith("gga")
    _, n, sig = _grid(5)
    q = sig / 4
    e1, v1, s1 = run_emu(emu, funs, n[None], sig[None] if gga else None)
    e2, v2, s2 = run_emu(emu, funs, np.array([n / 2, n / 2]), np.array([q, q, q]) if gga else None)
    np.testing.assert_allclose(e2, e1, rtol=1e-13)
    np.testing.assert_allclose(v2, np.array([v1[0], v1[0]]), rtol=1e-12)
    if gga:
        np.testing.assert_allclose(s2.sum(axis=0), 4 * s1[0], rtol=1e-12)
        np.testing.assert_allclose(s2[0], s2[2], rtol=1e-14)
        _, _, c1 = run_emu(emu, ("gga_c_pbe",), n[None], sig[None])
        _, _, c2 = run_emu(emu, ("gga_c_pbe",), np.array([n / 2, n / 2]), np.array([q, q, q]))
        np.testing.assert_allclose(c2, np.array([c1[0], 2 * c1[0], c1[0]]), rtol=1e-12)


@pytest.mark.parametrize("funs", [("lda_x", "lda_c_vwn"), ("lda_x", "lda_c_pw"), ("gga_x_pbe", "gga_c_pbe")])
def test_spin_flip_symmetry(emu, funs):
    """Swapping up and down leaves e unchanged and swaps vrho and vsigma_uu <-> vsigma_dd."""
    gga = funs[0].startswith("gga")
    rho, sigma = polarised_points(gga)
    e, vr, vs = run_emu(emu, funs, rho, sigma)
    ef, vrf, vsf = run_emu(emu, funs, rho[::-1], None if sigma is None else sigma[::-1])
    me, mr, ms = magnitudes(rho, sigma)     # the two orders of summation differ by rounding only
    assert np.all(np.abs(ef - e) <= 1e-14 * (np.abs(e) + me))
    assert np.all(np.abs(vrf[::-1] - vr) <= 1e-14 * (np.abs(vr) + mr))
    if gga:
        assert np.all(np.abs(vsf[::-1] - vs) <= 1e-14 * (np.abs(vs) + ms))


# ------------------------------------------------------------------ the fully polarised edge
def _edge_walk(n_up, sig_up):
    """rho_dn from 1e-6 rho_up down through the thresholds to 0 and to -1e-18 at fixed rho_up, sigma_uu."""
    rd = np.concatenate([n_up * 10.0 ** -np.arange(6.0, 31.0), [1e-20, 1e-25, 0.0, -1e-18]])
    rho = np.array([np.full(rd.size, n_up), rd])
    sigma = np.array([np.full(rd.size, sig_up), np.zeros(rd.size), np.zeros(rd.size)])
    return rho, sigma


@pytest.mark.parametrize("n_up,sig_up", [(1e-3, 1e-4), (0.1, 0.01), (1.0, 0.1)])
@pytest.mark.parametrize("funs", [("lda_x", "lda_c_pw"), ("lda_x", "lda_c_vwn"), ("gga_x_pbe", "gga_c_pbe")])
def test_fully_polarised_edge(emu, funs, n_up, sig_up):
    """Walking rho_dn to zero at a point with a majority gradient: e and vrho_up are continuous, every output is
    finite, and below the thresholds vrho_dn and vsigma_dd are the reference's screened values -- of order one, not
    the (1 - zeta)^(-1/3) of the correlation's phi(zeta) nor the rho_dn^(-4/3) of spin-resolved PBE exchange."""
    gga = funs[0].startswith("gga")
    rho, sigma = _edge_walk(n_up, sig_up)
    if not gga:
        sigma = None
    e, vr, vs = run_emu(emu, funs, rho, sigma)
    for x in (e, vr, vs):
        assert x is None or np.all(np.isfinite(x))
    # continuity of e and vrho_up as rho_dn -> 0, against the fully polarised value
    np.testing.assert_allclose(e, e[-2], rtol=1e-5)
    np.testing.assert_allclose(vr[0], vr[0, -2], rtol=1e-4)
    # below the thresholds the minority potentials are the screened reference values
    below = (rho[1] <= xr.DENS_THRESHOLD_SPIN) & (2 * rho[1] / rho.sum(axis=0) <= xr.ZETA_THRESHOLD)
    assert below.sum() >= 4
    re, rvr, rvs = reference(funs, rho[:, below], None if sigma is None else sigma[:, below])
    scale = abs(e[-2]) / n_up
    np.testing.assert_allclose(vr[:, below], rvr, rtol=1e-12, atol=1e-12 * scale)
    assert np.all(np.abs(rvr[1]) < 10 * scale)
    if gga:
        np.testing.assert_allclose(vs[:, below], rvs, rtol=1e-12, atol=1e-12 * scale / sig_up)
        assert np.all(np.abs(rvs[2]) < 10 * scale / sig_up * n_up)


@pytest.mark.parametrize("funs", [("lda_x", "lda_c_pw"), ("lda_x", "lda_c_vwn"), ("gga_x_pbe", "gga_c_pbe")])
def test_negative_minority_is_fully_polarised(emu, funs):
    """A negative spin density -- round-off, or a density mixer extrapolating next to an empty channel -- counts as an
    empty channel: e, vrho and vsigma equal those at rho_dn = 0 exactly, so zeta never leaves [-1, 1] (where zeta^4 and
    (1 + zeta)^p would grow without bound: zeta = 1999 at (1e-3, -9.99e-4))."""
    gga = funs[0].startswith("gga")
    up = np.array([1e-5, 0.1, 1e-3, 1e-3, 0.3])
    neg = np.array([-1e-6, -0.02, -9.99e-4, -1e-18, -0.299])
    sg = np.array([0.3 * sigma_unit(up), np.zeros(up.size), 0.2 * sigma_unit(-neg)]) if gga else None
    for flip in (False, True):
        rho_neg, rho_zero = np.array([up, neg]), np.array([up, np.zeros(up.size)])
        sig = sg
        if flip:
            rho_neg, rho_zero, sig = rho_neg[::-1], rho_zero[::-1], (None if sg is None else sg[::-1])
        got = run_emu(emu, funs, rho_neg, sig)
        ref = run_emu(emu, funs, rho_zero, sig)
        for g, r in zip(got, ref):
            if g is not None:
                assert np.all(np.isfinite(g))
                np.testing.assert_array_equal(g, r)
