"""UPF pseudopotentials on the host: the parser (dftk_b200.parse_upf and the oracle's restatement), the quadrature
weights, the oracle's radial transforms against the analytic HGH forms (test/PspUpf.jl of the reference) and against an
independent real-space quadrature, and the NLCC force of the oracle against finite differences of its energy."""
import math
import os
import numpy as np
import pytest

from oracle import psp_upf, nlcc
from oracle.psp_hgh import PspHgh
from oracle.basis import Element, Model, PlaneWaveBasis
from oracle.terms import Terms
from upf_data import UPF_DIR as UPF, product_psp, oracle_psp, upf_file

FILES = ["Si.pbe-hgh.upf", "Tl.pbe-d-hgh.upf", "Al_m.upf", "C_m.upf"]
PS = (0.01, 0.1, 0.2, 0.5, 1.0, 2.0, 5.0, 10.0)


_product = product_psp


@pytest.fixture(scope="module")
def oracle_psps():
    return {f: oracle_psp(f) for f in FILES}


# values copied by hand from the files: first PP_LOCAL, PP_DIJ[1,1], first PP_BETA.1, cutoff_radius_index of every β
PINS = {
    "Al_m.upf": dict(Zion=3, lmax=2, n=1842, vloc0=-7.6462870087E+00, dij00=-1.0884668374E+01, r0=0.0, beta0=3.3161462465E-10,
                     cut=[180] * 6, n_proj=2 * 1 + 2 * 3 + 2 * 5, core=True),
    "C_m.upf": dict(Zion=4, lmax=1, n=1232, vloc0=-1.4786243168E+01, dij00=1.3448417011E+01, r0=0.0, beta0=5.1637571996E-09,
                    cut=[132] * 4, n_proj=2 * 1 + 2 * 3, core=True),
    "Si.pbe-hgh.upf": dict(Zion=4, lmax=1, n=1141, vloc0=-2.704556847823059E+01, dij00=4.475870751000000E+00,
                           r0=6.513442611103688E-05, beta0=6.806137438802942E-04, cut=[871, 875, 885], n_proj=2 + 3,
                           core=False),
    "Tl.pbe-d-hgh.upf": dict(Zion=13, lmax=2, n=1281, vloc0=-1.313700894046930E+01, dij00=3.595085084500000E+00,
                             r0=1.125780204388292E-05, beta0=9.210860659946899E-05, cut=[1025, 1029, 1037, 1039, 1007, 1011],
                             n_proj=2 + 2 * 3 + 2 * 5, core=False),
}


@pytest.mark.parametrize("name", FILES)
def test_parser_pins(name, oracle_psps):
    pin = PINS[name]
    for psp in (_product(name), oracle_psps[name]):
        assert psp.Zion == pin["Zion"] and psp.lmax == pin["lmax"]
        assert len(psp.rgrid) == pin["n"] and len(psp.vloc) == pin["n"]
        assert psp.vloc[0] == pin["vloc0"] / 2
        assert psp.h[0][0, 0] == pin["dij00"] * 2
        assert psp.r2_projs[0][0][0] == pin["r0"] * (pin["beta0"] / 2)
        cuts = [len(f) for fl in psp.r2_projs for f in fl]
        assert sorted(cuts) == sorted(pin["cut"])
        assert psp.has_core_density == pin["core"]
    prod = _product(name)
    assert prod.count_n_proj() == pin["n_proj"] == oracle_psps[name].n_proj()
    assert prod.rcut == prod.rgrid[-1]
    assert prod.identifier.endswith(name)
    for l in range(prod.lmax + 1):
        np.testing.assert_array_equal(prod.h[l], oracle_psps[name].h[l])
        assert prod.h[l].shape == (len(prod.r2_projs[l]),) * 2


def test_taumod_is_kept():
    psp = _product("Al_m.upf")
    assert np.any(psp.r2_taucore != 0) and psp.has_valence_density


def _synthetic(**header):
    attrs = dict(element="Si", pseudo_type="NC", has_so="F", has_gipaw="F", z_valence="4.0", l_max="0", mesh_size="5")
    attrs.update(header)
    hd = " ".join(f'{k}="{v}"' for k, v in attrs.items())
    return (f'<UPF version="2.0.1">\n<PP_HEADER {hd}/>\n<PP_MESH><PP_R>0.0 0.1 0.2 0.3 0.4</PP_R>'
            f'<PP_RAB>0.1 0.1 0.1 0.1 0.1</PP_RAB></PP_MESH>\n<PP_LOCAL>-1 -1 -1 -1 -1</PP_LOCAL>\n'
            f'<PP_NONLOCAL><PP_BETA.1 angular_momentum="0" cutoff_radius_index="3">1 1 1 0 0</PP_BETA.1>'
            f'<PP_DIJ>0.5</PP_DIJ></PP_NONLOCAL>\n</UPF>\n')


@pytest.mark.parametrize("header,what", [
    (dict(pseudo_type="US"), "ultrasoft"), (dict(pseudo_type="USPP"), "ultrasoft"),
    (dict(pseudo_type="PAW"), "projector-augmented"), (dict(pseudo_type="SL"), "semilocal"),
    (dict(pseudo_type="1/r"), "Coulomb"), (dict(has_so="T"), "spin-orbit"), (dict(has_gipaw="T"), "gipaw"),
    (dict(l_max="4"), "l_max")])
def test_unsupported_headers_are_rejected(header, what):
    from dftk_b200 import parse_upf
    parse_upf(_synthetic(), "ok")                      # the synthetic file itself is accepted
    psp_upf.PspUpf(_synthetic())
    with pytest.raises(ValueError, match=what):
        parse_upf(_synthetic(**header), "bad")
    with pytest.raises(ValueError):
        psp_upf.PspUpf(_synthetic(**header))


def test_upf_v1_is_rejected():
    from dftk_b200 import parse_upf
    v1 = "<PP_INFO>\n old format\n</PP_INFO>\n<PP_HEADER>\n   0   Version Number\n</PP_HEADER>\n"
    with pytest.raises(ValueError, match="version 2"):
        parse_upf(v1)
    with pytest.raises(ValueError):
        psp_upf.PspUpf(v1)


def test_load_psp_dispatches_on_extension(tmp_path):
    from dftk_b200 import load_psp, PspHgh as PH, PspUpf as PU
    assert isinstance(load_psp(os.path.join(UPF, "Si-q4.gth")), PH)
    psp = load_psp(upf_file("Si.pbe-hgh.upf", tmp_path))
    assert isinstance(psp, PU) and psp.identifier.endswith("Si.pbe-hgh.upf")
    np.testing.assert_array_equal(psp.vloc, _product("Si.pbe-hgh.upf").vloc)
    assert isinstance(load_psp("Si", "pbe"), PH)       # the built-in tables are unchanged


@pytest.mark.parametrize("name", FILES)
def test_quadrature_weights_match_oracle(name, oracle_psps):
    """Product and oracle weights on every truncation length the transforms use (uniform Al/C and log Si/Tl meshes,
    with even and odd interval counts), and the choice of rule with Julia's ≈ (rtol √eps, atol 0)."""
    prod, orc = _product(name), oracle_psps[name]
    assert prod._uniform == psp_upf.is_uniform(orc.rgrid) == name.endswith("_m.upf")
    lengths = {len(prod.rgrid), len(prod.rgrid) - 1} | {len(f) for fl in prod.r2_projs for f in fl}
    for n in lengths:
        np.testing.assert_allclose(prod.weights(n), psp_upf.psp_quadrature_weights(orc.rgrid, n), rtol=1e-14, atol=0)
    assert {(n - 1) % 2 for n in lengths} == {0, 1}
    # numpy's isclose defaults would call the log mesh uniform; the reference's rule does not
    if name == "Tl.pbe-d-hgh.upf":
        r = orc.rgrid
        assert np.isclose(r[1] - r[0], r[2] - r[1]) and not psp_upf.is_uniform(r)


@pytest.mark.parametrize("upf,gth", [("Si.pbe-hgh.upf", "Si-q4.gth"), ("Tl.pbe-d-hgh.upf", "Tl-q13.gth")])
def test_oracle_upf_matches_analytic_hgh(upf, gth, oracle_psps):
    """test/PspUpf.jl: local 1e-3, projectors 1e-5, energy correction 1e-3."""
    u = oracle_psps[upf]
    g = PspHgh.parse(open(os.path.join(UPF, gth)).read())
    p = np.array(PS)
    np.testing.assert_allclose(u.eval_local_fourier(p), g.eval_local_fourier(p), rtol=1e-3, atol=1e-3)
    assert u.lmax == g.lmax
    for l in range(u.lmax + 1):
        assert u.n_proj_radial(l) == g.n_proj_radial(l)
        np.testing.assert_allclose(u.h[l], g.h[l], rtol=1e-8)
        for i in range(1, u.n_proj_radial(l) + 1):
            np.testing.assert_allclose(u.eval_projector_fourier(i, l, p), g.eval_projector_fourier(i, l, p), rtol=1e-5,
                                       atol=1e-5)
    assert u.energy_correction() == pytest.approx(g.energy_correction(), rel=1e-3, abs=1e-3)
    assert _product(upf).eval_psp_energy_correction() == pytest.approx(u.energy_correction(), rel=1e-14)


def _fine_integral(f, a, b, p, l):
    """4π/p^l ∫_a^b r² f(r) j_l(p r) dr on a dense uniform grid of the interpolated real-space function."""
    from scipy.special import spherical_jn
    from scipy.integrate import simpson
    r = np.linspace(a, b, 400001)
    return 4 * math.pi * simpson(r ** 2 * f(r) * spherical_jn(l, p * r), x=r) / p ** l


@pytest.mark.parametrize("name", FILES)
def test_real_and_fourier_forms_are_consistent(name, oracle_psps):
    """test/PspUpf.jl 'consistent in real and Fourier space' (atol = rtol = 1e-2), for the local potential, every
    projector and the valence and core densities."""
    psp = oracle_psps[name]
    r = psp.rgrid
    a = r[1] if r[0] == 0 else r[0]
    for p in PS:
        ref = _fine_integral(lambda x: psp.eval_local_real(x) + psp.Zion / x, a, r[-1], p, 0) - 4 * math.pi * psp.Zion / p ** 2
        assert ref == pytest.approx(psp.eval_local_fourier([p])[0], rel=1e-2, abs=1e-2)
        for l in range(psp.lmax + 1):
            for i in range(1, psp.n_proj_radial(l) + 1):
                cut = len(psp.r2_projs[l][i - 1])
                ref = _fine_integral(lambda x: psp.eval_projector_real(i, l, x), a, r[cut - 1], p, l)
                assert ref == pytest.approx(psp.eval_projector_fourier(i, l, [p])[0], rel=1e-2, abs=1e-2)
        for kind in ("valence", "core"):
            ref = _fine_integral(getattr(psp, f"eval_{kind}_density_real"), a, r[-1], p, 0)
            assert ref == pytest.approx(getattr(psp, f"eval_{kind}_density_fourier")([p])[0], rel=1e-2, abs=1e-2)


@pytest.mark.parametrize("name", ["Si.pbe-hgh.upf", "Al_m.upf", "C_m.upf"])
def test_pseudo_valence_density_integrates_to_zion(name, oracle_psps):
    psp = oracle_psps[name]
    assert psp.has_valence_density
    assert psp.eval_valence_density_fourier([0.0])[0] == pytest.approx(psp.Zion, abs=1e-5)
    prod = _product(name)
    assert 4 * math.pi * float(np.sum(prod.weights(len(prod.rgrid)) * prod.r2_rhoion)) == pytest.approx(psp.Zion, abs=1e-5)


# ------------------------------------------------------------------ NLCC forces of the oracle
A_DIAMOND = 6.74


def _carbon(positions, psp):
    lat = A_DIAMOND / 2 * np.array([[0.0, 1, 1], [1, 0, 1], [1, 1, 0]])
    c = Element("C", psp)
    return Model(lat, [c, c], positions, functionals=("lda_x", "lda_c_pw"), symmetries=False)


@pytest.fixture(scope="module")
def displaced_carbon(oracle_psps):
    psp = oracle_psps["C_m.upf"]
    pos = [np.ones(3) / 8 + np.array([0.012, -0.006, 0.004]), -np.ones(3) / 8]
    model = _carbon(pos, psp)
    basis = PlaneWaveBasis(model, Ecut=10, kgrid=(1, 1, 1))
    res = nlcc.self_consistent_field(basis, tol=1e-10, maxiter=80)
    assert res["converged"]
    return psp, model, basis, res


def test_nlcc_force_matches_xc_energy_derivative(displaced_carbon):
    """With ψ, occupation and ρ held fixed only ρcore moves with the atom: the Xc force is -dE_xc/dR exactly."""
    psp, model, basis, res = displaced_carbon
    _, parts = nlcc.compute_forces(basis, res["psi"], res["occupation"], res["rho"])
    assert "Xc" in parts and np.linalg.norm(parts["Xc"][0]) > 1e-3
    direction = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    eps = 1e-5

    def e_xc(e):
        pos = [model.positions[0] + e * direction, model.positions[1]]
        mb = PlaneWaveBasis(_carbon(pos, psp), Ecut=10, fft_size=basis.fft_size, kcoords=basis.kcoords_global,
                            kweights=basis.kweights_global)
        return nlcc.energy_hamiltonian(mb, Terms(mb), res["psi"], res["occupation"], res["rho"], res["eigenvalues"],
                                       res["eF"], only_energy=True, rhocore=nlcc.core_density(mb))[0]["Xc"]
    fd = -(e_xc(eps) - e_xc(-eps)) / (2 * eps)
    assert float(direction @ parts["Xc"][0]) == pytest.approx(fd, abs=1e-7)


def test_nlcc_total_force_is_energy_derivative(displaced_carbon):
    """-dE_total/dx of re-converged SCFs (test/forces.jl:59-88) equals the total force, the NLCC term included."""
    psp, model, basis, res = displaced_carbon
    total, parts = nlcc.compute_forces(basis, res["psi"], res["occupation"], res["rho"])
    direction = np.array([0.0, 0.0, 1.0])
    eps = 1e-4

    def etot(e):
        pos = [model.positions[0] + e * direction, model.positions[1]]
        mb = PlaneWaveBasis(_carbon(pos, psp), Ecut=10, fft_size=basis.fft_size, kcoords=basis.kcoords_global,
                            kweights=basis.kweights_global)
        r = nlcc.self_consistent_field(mb, rho=res["rho"], tol=1e-10, maxiter=80)
        assert r["converged"]
        return r["energies"]["total"]
    fd = -(etot(eps) - etot(-eps)) / (2 * eps)
    hf = float(direction @ total[0])
    without_xc = float(direction @ (total[0] - parts["Xc"][0]))
    assert hf == pytest.approx(fd, abs=1e-6)
    assert abs(without_xc - fd) > 100 * abs(hf - fd)     # the NLCC term is what closes the gap
