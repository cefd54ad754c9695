"""The Teter-Pade and Perdew-Zunger LDAs and the PBEsol, revPBE and RPBE GGAs of the XC kernel (xc_core.cuh, host
build of tests/hostemu/emu.cu): against the extended-precision reference of tests/xc_reference_families.py over the
sweep of test_xc_reference, against identities, against the oracle's restatement (tests/xc_oracle_families.py), and the
reference's iron LDA SCF (test/iron_lda.jl) on the oracle against ABINIT."""
import ctypes
import json
import math
import os
import numpy as np
import pytest

import xc_reference as xr
import xc_reference_families as xrf
import xc_oracle_families
from test_xc_reference import (emu, polarised_points, unpolarised_points, magnitudes, assert_close,  # noqa: F401
                               sigma_unit, _grid, _p)

# libxc symbol -> mask bit of the kernel, every functional it carries
MASK = {"lda_x": 1, "lda_c_vwn": 2, "lda_c_pw": 4, "gga_x_pbe": 8, "gga_c_pbe": 16, "lda_xc_teter93": 32,
        "lda_c_pz": 64, "gga_x_pbe_sol": 128, "gga_c_pbe_sol": 256, "gga_x_pbe_r": 512, "gga_x_rpbe": 1024}
NEW_X = ("gga_x_pbe_sol", "gga_x_pbe_r", "gga_x_rpbe")
# the functional sets users run: PBEsol, revPBE, RPBE, Teter-Pade, Slater + Perdew-Zunger
SETS = [("gga_x_pbe_sol", "gga_c_pbe_sol"), ("gga_x_pbe_r", "gga_c_pbe"), ("gga_x_rpbe", "gga_c_pbe"),
        ("lda_xc_teter93",), ("lda_x", "lda_c_pz")]
SET_IDS = ["pbesol", "revpbe", "rpbe", "teter93", "pz"]


def run_emu(lib, funs, rho, sigma=None):
    """test_xc_reference.run_emu over every mask bit of the kernel."""
    rho = np.ascontiguousarray(rho, dtype=float)
    n_spin, N = rho.shape
    gga = any(f.startswith("gga") for f in funs)
    nsig = (1 if n_spin == 1 else 3) if gga else 0
    sg = np.ascontiguousarray(sigma if gga else np.zeros((1, N)), dtype=float)
    e, vr, vs = np.zeros(N), np.zeros((n_spin, N)), np.zeros((max(nsig, 1), N))
    mask = sum(MASK[f] for f in funs)
    assert lib.emu_xc(mask, n_spin, int(gga), ctypes.c_int64(N), _p(rho), _p(sg), _p(e), _p(vr), _p(vs)) == 0
    return e, vr, (vs if gga else None)


_REF_CACHE = {}


def reference(funs, rho, sigma):
    key = (funs, rho.tobytes(), None if sigma is None else sigma.tobytes())
    if key not in _REF_CACHE:
        N = rho.shape[1]
        e, vr, vs = np.zeros(N), np.zeros(rho.shape), None if sigma is None else np.zeros(sigma.shape)
        for i in range(N):
            ee, r, s = xrf.evaluate(funs, rho[:, i], () if sigma is None else sigma[:, i])
            e[i] = float(ee)
            vr[:, i] = [float(x) for x in r]
            if sigma is not None:
                vs[:, i] = [float(x) for x in s]
        _REF_CACHE[key] = (e, vr, vs)
    return _REF_CACHE[key]


def sweep_points(functional, n_spin):
    return (unpolarised_points if n_spin == 1 else polarised_points)(functional.startswith("gga"))


# ------------------------------------------------------------------ the sweep
@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("functional", xrf.FUNCTIONALS)
def test_sweep_matches_reference(emu, functional, n_spin):
    """Each new functional alone over the sweep of test_xc_reference (log density grid, every zeta to the fully
    polarised edge, every reduced gradient, negative minorities) within its bound, against the mpmath reference."""
    rho, sigma = sweep_points(functional, n_spin)
    e, vr, vs = run_emu(emu, (functional,), rho, sigma)
    re, rvr, rvs = reference((functional,), rho, sigma)
    me, mr, ms = magnitudes(rho, sigma)
    assert_close(e, re, me, "e", rho, sigma)
    assert_close(vr, rvr, mr[None, :], "vrho", rho, sigma)
    if sigma is not None:
        assert_close(vs, rvs, ms[None, :], "vsigma", rho, sigma)


@pytest.mark.parametrize("funs", SETS, ids=SET_IDS)
def test_combined_functionals_are_the_sum(emu, funs):
    gga = funs[0].startswith("gga")
    rho, sigma = polarised_points(gga)
    both = run_emu(emu, funs, rho, sigma)
    parts = [run_emu(emu, (f,), rho, sigma) for f in funs]
    for k in range(3 if gga else 2):
        total = sum(p[k] for p in parts)
        np.testing.assert_allclose(both[k], total, rtol=1e-14, atol=1e-14 * np.abs(total).max())


# ------------------------------------------------------------------ identities
@pytest.mark.parametrize("functional", NEW_X)
def test_exchange_spin_scaling(emu, functional):
    """E_x[rho_up, rho_dn] = (E_x[2 rho_up] + E_x[2 rho_dn]) / 2 with each sigma scaled by 4."""
    rng, n, sig = _grid(1)
    z = rng.uniform(-1, 1, n.size)
    ru, rd = n * (1 + z) / 2, n * (1 - z) / 2
    suu, sdd = sig * (1 + z) ** 2 / 4, sig * (1 - z) ** 2 / 4
    e, vr, vs = run_emu(emu, (functional,), np.array([ru, rd]), np.array([suu, np.sqrt(suu * sdd), sdd]))
    eu, vu, su = run_emu(emu, (functional,), (2 * ru)[None], (4 * suu)[None])
    ed, vd, sd = run_emu(emu, (functional,), (2 * rd)[None], (4 * sdd)[None])
    np.testing.assert_allclose(e, (eu + ed) / 2, rtol=1e-13)
    np.testing.assert_allclose(vr, np.array([vu[0], vd[0]]), rtol=1e-13)
    # RPBE's vsigma ~ exp(-mu s^2 / kappa) reaches subnormal values at large s, where only an absolute bound holds
    np.testing.assert_allclose(vs[[0, 2]], 2 * np.array([su[0], sd[0]]), rtol=1e-13, atol=1e-300)
    assert np.all(vs[1] == 0.0)


@pytest.mark.parametrize("functional", NEW_X)
def test_exchange_uniform_scaling(emu, functional):
    """e_x(lambda^3 n, lambda^8 sigma) = lambda^4 e_x(n, sigma)."""
    _, n, sig = _grid(2)
    e0, _, _ = run_emu(emu, (functional,), n[None], sig[None])
    for lam in (1e-2, 0.37, 5.0, 40.0):
        e1, _, _ = run_emu(emu, (functional,), (lam ** 3 * n)[None], (lam ** 8 * sig)[None])
        np.testing.assert_allclose(e1, lam ** 4 * e0, rtol=1e-13)


def _spin_grid(n_spin, seed, N=200):
    rng, n, _ = _grid(seed, N)
    z = rng.uniform(-0.99, 0.99, n.size) if n_spin == 2 else np.zeros(n.size)
    rho = np.array([n * (1 + z) / 2, n * (1 - z) / 2]) if n_spin == 2 else n[None]
    return n, z, rho


@pytest.mark.parametrize("n_spin", [1, 2])
def test_gga_reduces_to_lda_at_zero_gradient(emu, n_spin):
    """At sigma = 0 every new exchange is Dirac exchange, and PBEsol correlation is PBE correlation, i.e. PW92-mod."""
    n, _, rho = _spin_grid(n_spin, 3)
    sigma = np.zeros((3 if n_spin == 2 else 1, n.size))
    lx, lvx, _ = run_emu(emu, ("lda_x",), rho)
    for f in NEW_X:
        ex, vx, _ = run_emu(emu, (f,), rho, sigma)
        np.testing.assert_allclose(ex, lx, rtol=1e-13)
        np.testing.assert_allclose(vx, lvx, rtol=1e-13)
    ec, vc, _ = run_emu(emu, ("gga_c_pbe_sol",), rho, sigma)
    ep, vp, _ = run_emu(emu, ("gga_c_pbe",), rho, sigma)
    np.testing.assert_allclose(ec, ep, rtol=1e-13)
    np.testing.assert_allclose(vc, vp, rtol=1e-13)


@pytest.mark.parametrize("functional,mu", [("gga_x_pbe_sol", 10 / 81),
                                           ("gga_x_pbe_r", 0.06672455060314922 * math.pi ** 2 / 3),
                                           ("gga_x_rpbe", 0.06672455060314922 * math.pi ** 2 / 3)])
def test_exchange_enhancement_limits(emu, functional, mu):
    """F_x - 1 = mu s^2 at small s (the gradient expansion each functional is built on: mu = 10/81 for PBEsol) and
    F_x -> 1 + kappa at large s."""
    kappa = 1.245 if functional == "gga_x_pbe_r" else 0.804
    n = 10.0 ** np.linspace(-6, 3, 10)
    lx, _, _ = run_emu(emu, ("lda_x",), n[None])
    for s, check in ((1e-4, lambda fx: np.testing.assert_allclose(fx - 1, mu * 1e-8, rtol=1e-6)),
                     (1e3, lambda fx: np.testing.assert_allclose(fx, 1 + kappa, rtol=1e-5))):
        ex, _, _ = run_emu(emu, (functional,), n[None], (s * s * sigma_unit(n))[None])
        check(ex / lx)


@pytest.mark.parametrize("zeta", [0.0, 0.6])
def test_pbe_sol_gradient_correction_small_t(emu, zeta):
    """The PBEsol correlation's gradient correction H tends to beta phi^3 t^2 (beta = 0.046) as t -> 0."""
    n = 10.0 ** np.linspace(-4, 2, 13)
    phi = ((1 + zeta) ** (2 / 3) + (1 - zeta) ** (2 / 3)) / 2
    t2 = 1e-6
    sig = t2 * 4 * phi ** 2 * (4 * (3 * math.pi ** 2 * n) ** (1 / 3) / math.pi) * n ** 2
    rho = np.array([n * (1 + zeta) / 2, n * (1 - zeta) / 2])
    z0 = np.zeros_like(n)
    e, _, _ = run_emu(emu, ("gga_c_pbe_sol",), rho, np.array([sig / 4, sig / 4, sig / 4]))
    e0, _, _ = run_emu(emu, ("gga_c_pbe_sol",), rho, np.array([z0, z0, z0]))
    np.testing.assert_allclose((e - e0) / n, 0.046 * phi ** 3 * t2, rtol=1e-4)


@pytest.mark.parametrize("funs", SETS, ids=SET_IDS)
def test_spin_paths_agree_at_zeta_zero(emu, funs):
    """n_spin = 2 at rho_up = rho_dn = n / 2 reproduces n_spin = 1 (vsigma through sigma = sigma_uu + 2 sigma_ud +
    sigma_dd, every sigma_st = sigma / 4)."""
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


@pytest.mark.parametrize("funs", SETS, ids=SET_IDS)
def test_spin_flip_symmetry(emu, funs):
    """Swapping up and down leaves e unchanged and swaps vrho and vsigma_uu <-> vsigma_dd."""
    gga = funs[0].startswith("gga")
    rho, sigma = polarised_points(gga)
    e, vr, vs = run_emu(emu, funs, rho, sigma)
    ef, vrf, vsf = run_emu(emu, funs, rho[::-1], None if sigma is None else sigma[::-1])
    me, mr, ms = magnitudes(rho, sigma)
    assert np.all(np.abs(ef - e) <= 1e-14 * (np.abs(e) + me))
    assert np.all(np.abs(vrf[::-1] - vr) <= 1e-14 * (np.abs(vr) + mr))
    if gga:
        assert np.all(np.abs(vsf[::-1] - vs) <= 1e-14 * (np.abs(vs) + ms))


def _lda_at(rs, zeta):
    n = 3 / (4 * math.pi * rs ** 3)
    return n, np.array([n * (1 + zeta) / 2, n * (1 - zeta) / 2])


@pytest.mark.parametrize("zeta", [0.0, 0.5, 1.0])
def test_teter_pade_is_close_to_slater_pw92(emu, zeta):
    """Teter-Pade is a fit to exchange plus the Ceperley-Alder correlation, so over rs 0.1 to 50 it stays within 2e-3
    of lda_x + lda_c_pw (largest measured gap 9.9e-4)."""
    _, rho = _lda_at(10.0 ** np.linspace(-1, math.log10(50), 60), zeta)
    et, _, _ = run_emu(emu, ("lda_xc_teter93",), rho)
    ep, _, _ = run_emu(emu, ("lda_x", "lda_c_pw"), rho)
    assert np.all(np.abs(et - ep) <= 2e-3 * np.abs(ep))


@pytest.mark.parametrize("zeta", [0.0, 1.0])
def test_perdew_zunger_is_close_to_pw92(emu, zeta):
    """Perdew-Zunger and PW92 fit the same Ceperley-Alder data: within 2 % of each other over rs 0.1 to 50 in the
    paramagnetic and ferromagnetic limits (largest measured gap 1.2 %)."""
    _, rho = _lda_at(10.0 ** np.linspace(-1, math.log10(50), 60), zeta)
    ez, _, _ = run_emu(emu, ("lda_c_pz",), rho)
    ep, _, _ = run_emu(emu, ("lda_c_pw",), rho)
    assert np.all(np.abs(ez - ep) <= 0.02 * np.abs(ep))


# ------------------------------------------------------------------ the oracle's restatement
@pytest.mark.parametrize("n_spin", [1, 2])
@pytest.mark.parametrize("functional", xrf.FUNCTIONALS)
def test_oracle_matches_host_build(emu, functional, n_spin):
    """tests/xc_oracle_families.py (the oracle's NumPy duals) against the kernel's host build over the sweep, within
    the sweep's bound."""
    rho, sigma = sweep_points(functional, n_spin)
    e, vr, vs = run_emu(emu, (functional,), rho, sigma)
    o = xc_oracle_families.evaluate([functional], rho, sigma)
    me, mr, ms = magnitudes(rho, sigma)
    assert_close(o["e"], e, me, "e", rho, sigma)
    assert_close(o["Vrho"], vr, mr[None, :], "vrho", rho, sigma)
    if sigma is not None:
        assert_close(o["Vsigma"], vs, ms[None, :], "vsigma", rho, sigma)


def test_oracle_keeps_its_own_functionals():
    """The extension hands the oracle's functionals to it unchanged, and adds a new one to them term by term."""
    import oracle.xc as ox
    rho, sigma = polarised_points(True)
    for funs in (["gga_x_pbe", "gga_c_pbe"], ["lda_x", "lda_c_pw"]):
        a, b = ox.evaluate(funs, rho, sigma), xc_oracle_families.evaluate(funs, rho, sigma)
        for k in ("e", "Vrho", "Vsigma"):
            if a[k] is None:
                assert b[k] is None
            else:
                np.testing.assert_array_equal(a[k], b[k])
    both = xc_oracle_families.evaluate(["gga_x_rpbe", "gga_c_pbe"], rho, sigma)
    x = xc_oracle_families.evaluate(["gga_x_rpbe"], rho, sigma)
    c = ox.evaluate(["gga_c_pbe"], rho, sigma)
    for k in ("e", "Vrho", "Vsigma"):
        np.testing.assert_allclose(both[k], x[k] + c[k], rtol=1e-14, atol=1e-14 * np.abs(x[k] + c[k]).max())
    with pytest.raises(NotImplementedError):
        xc_oracle_families.evaluate(["gga_x_b88"], rho, sigma)


# ------------------------------------------------------------------ iron LDA against ABINIT
# the reference's GTH-PADE iron and the ABINIT numbers of its test/iron_lda.jl (tests/golden/iron_lda/README.md)
IRON_LDA_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "iron_lda")
IRON_LDA_PSP = os.path.join(IRON_LDA_DIR, "Fe-q8.hgh")


def iron_lda_reference():
    with open(os.path.join(IRON_LDA_DIR, "abinit.json")) as fh:
        return json.load(fh)


def iron_lda_psp_text():
    with open(IRON_LDA_PSP) as fh:
        return fh.read()


IRON_LATTICE = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)


def assert_iron_lda_matches_abinit(kpoints, eigenvalues, total, ref):
    """E_tot and every (k, spin) block's lowest 8 eigenvalues to the reference's tolerance.  The irreducible k-points
    come from an orbit search, not spglib: blocks are matched to ABINIT's by their spectra, each used once."""
    tol = ref["tolerance"]
    assert abs(total - ref["energy_total"]) < tol
    used = set()
    for ik, kpt in enumerate(kpoints):
        d = [np.abs(np.array(eigenvalues[ik][:8]) - np.array(r)).max() for r in ref["eigenvalues"]]
        j = int(np.argmin(d))
        assert d[j] < tol and (j < 6) == (kpt.spin == 0), (ik, j, d[j])
        used.add(j)
    assert used == set(range(12))


def test_iron_lda_scf_vs_abinit_on_oracle(monkeypatch):
    # reference: test/iron_lda.jl (bcc Fe, GTH-PADE-q8, lda_xc_teter93, collinear spin, Fermi-Dirac T = 0.01, Ecut 15,
    # fft 20, shifted 4x4x4 k-grid; ABINIT eigenvalues and E_tot to 5e-6) -- pins the Teter-Pade constants
    from oracle.psp_hgh import PspHgh
    from oracle.basis import Element, Model, PlaneWaveBasis
    from oracle.terms import guess_density
    from oracle import scf
    xc_oracle_families.install(monkeypatch)
    ref = iron_lda_reference()
    psp = PspHgh.parse(iron_lda_psp_text())
    psp.Z = 26                       # the file carries only the valence charge
    m = Model(IRON_LATTICE, [Element("Fe", psp)], [np.zeros(3)],
              functionals=("lda_xc_teter93",), temperature=0.01, magnetic_moments=[4.0])
    b = PlaneWaveBasis(m, 15, kgrid=(4, 4, 4), kshift=(0.5, 0.5, 0.5), fft_size=(20, 20, 20))
    assert len(b.kpoints) == 12 and m.n_electrons == 8

    def conv(info):
        h = info["history_Etot"]
        return len(h) > 1 and abs(h[-1] - h[-2]) < 1e-10
    res = scf.self_consistent_field(b, rho=guess_density(b, [4.0]), mixing="kerker",
                                    nbandsalg=scf.AdaptiveBands(m, n_bands_converge=8), is_converged=conv)
    assert_iron_lda_matches_abinit(b.kpoints, res["eigenvalues"], res["energies"]["total"], ref)
