"""Cold and Methfessel-Paxton smearing and energy-cutoff smearing on the device, against the oracle (extended by
tests/smearing_oracle.py): SCF energies, Fermi level, eigenvalues, density and forces of the C4-shape aluminium cell;
the reference's energy-cutoff smearing test (test/energy_cutoff_smearing.jl); Hψ with a blown-up kinetic table on the
large single-block and the batched k-grid paths; SCF and direct minimisation with BlowupCHV; the slab path on 2 GPUs."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import smearing_oracle as so
from silicon import LATTICE, POSITIONS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _compare_scf(res, ores, basis, ob, n_atoms, n_cmp):
    """The tolerances of test_gpu_scf.py."""
    assert abs(res["energies"].total - ores["energies"]["total"]) < 1e-8 * max(1, n_atoms) + 1e-9
    for ik, kpt in enumerate(basis.kpoints):
        jk = [j for j, ok in enumerate(ob.kpoints) if ok.spin == kpt.spin and np.allclose(ok.coordinate, kpt.coordinate)][0]
        np.testing.assert_allclose(res["eigenvalues"][ik][:n_cmp], ores["eigenvalues"][jk][:n_cmp], atol=1e-6)
    drho = res["rho"].cpu().numpy() - ores["rho"]
    assert np.linalg.norm(drho) * math.sqrt(basis.dvol) < 1e-7


@pytest.mark.parametrize("smearing", ["MarzariVanderbilt", ("MethfesselPaxton", 1)], ids=str)
def test_aluminium_pbe_cold_smearing_matches_oracle(smearing):
    """BASELINE config C4 shape (Al fcc 4-atom PBE, Kerker mixing, Ecut 7, 2³ k) with the two-stage Fermi search."""
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle import scf as oscf, forces as oforces
    a = 7.65339
    lat = a * np.eye(3)
    pos = [[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]]
    Al = dftk.ElementPsp("Al", functional="pbe")
    model = dftk.model_DFT(lat, [Al] * 4, pos, functionals=dftk.PBE(), temperature=0.01, smearing=smearing)
    basis = dftk.PlaneWaveBasis(model, Ecut=7, kgrid=(2, 2, 2))
    res = dftk.self_consistent_field(basis, tol=1e-9, mixing=dftk.KerkerMixing())
    assert res["converged"]
    om = Model(lat, [Element("Al", functional="pbe")] * 4, pos, functionals=("gga_x_pbe", "gga_c_pbe"),
               temperature=0.01, smearing=smearing)
    ob = OBasis(om, 7, kgrid=(2, 2, 2))
    with so.extended():
        ores = oscf.self_consistent_field(ob, tol=1e-9, mixing="kerker")
    assert abs(res["eF"] - ores["eF"]) < 1e-6
    assert abs(res["energies"]["Entropy"]) > 1e-6
    assert abs(res["energies"]["Entropy"] - ores["energies"]["Entropy"]) < 1e-7
    _compare_scf(res, ores, basis, ob, 4, 6)
    ototal, _ = oforces.compute_forces(ob, ores["psi"], ores["occupation"], ores["rho"])
    np.testing.assert_allclose(np.array(dftk.compute_forces_cart(res)),
                               np.array([np.linalg.inv(lat).T @ f for f in ototal]), atol=1e-7)


def _si_lda(**kw):
    import dftk_b200 as dftk
    Si = dftk.ElementPsp("Si")
    return dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), **kw)


def test_energy_cutoff_smearing_regularises_the_band():
    """test/energy_cutoff_smearing.jl: the lowest silicon band at Ecut 5 has a discontinuity between X and U; with a
    blown-up kinetic term the same band is C², so ‖∂²λ_std‖ / ‖∂²λ_blowup‖ > 1e4 on 100 k-points across it."""
    import dftk_b200 as dftk
    basis_std = dftk.PlaneWaveBasis(_si_lda(), Ecut=5, kgrid=(3, 3, 3))
    scfres = dftk.self_consistent_field(basis_std, tol=1e-10)
    assert scfres["converged"]
    k0, k1 = np.array([0.5274, 0.0548, 0.5274]), np.array([0.5287, 0.0573, 0.5287])
    kcoords = [(1 - x) * k0 + x * k1 for x in np.linspace(0, 1, 100)]
    dk = np.abs(kcoords[1] - kcoords[0]).sum()

    def band(blowup):
        model = _si_lda(kinetic_blowup=blowup)
        basis = dftk.PlaneWaveBasis(model, Ecut=5, kgrid=dftk.ExplicitKpoints(kcoords), fft_size=basis_std.fft_size)
        _, ham = dftk.energy_hamiltonian(basis, None, None, rho=scfres["rho"])
        res = dftk.diagonalize_all_kblocks(dftk.lobpcg_hyper, ham, 4, tol=1e-9)
        assert res["converged"]
        lam = np.array([l[0] for l in res["λ"]])
        return (lam[2:] - 2 * lam[1:-1] + lam[:-2]) / dk ** 2

    d2_std = np.linalg.norm(band(None))
    for blowup in (dftk.BlowupCHV(), dftk.BlowupAbinit()):
        assert d2_std / np.linalg.norm(band(blowup)) > 1e4, blowup


def _oracle_blocks(model_kw, basis, rho, blowup, kcoords, kweights):
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle.terms import Terms, energy_hamiltonian
    om = Model(basis.model.lattice, [Element("Si")] * len(basis.model.atoms), basis.model.positions, symmetries=False,
               **model_kw)
    with so.extended(blowup):
        ob = OBasis(om, basis.Ecut, fft_size=basis.fft_size, kcoords=kcoords, kweights=kweights)
        _, blocks = energy_hamiltonian(ob, Terms(ob), None, None, rho)
    return ob, blocks


def _hpsi_check(basis, ham, oblocks, apply):
    g = torch.Generator(device="cpu").manual_seed(5)
    psis = [torch.view_as_complex(torch.randn(6, kpt.n_G, 2, generator=g, dtype=torch.float64)).to("cuda")
            for kpt in basis.kpoints]
    outs = apply(psis)
    for ik, (psi, out) in enumerate(zip(psis, outs)):
        ref = oblocks[ik].matmul(psi.cpu().numpy().T).T
        err = np.abs(out.cpu().numpy() - ref).max() / np.abs(ref).max()
        assert err < 1e-12, (ik, err)
    return outs


def test_hpsi_with_blown_up_kinetic_table_matches_oracle():
    """Hψ with BlowupCHV / BlowupAbinit tables: the large single block (Γ supercell, folded nonlocal) and the batched
    small blocks of a k-grid (dftk_b200_apply_h_multi) against the oracle's Hψ at 1e-12."""
    import dftk_b200 as dftk
    from dftk_b200 import device as dev
    rep = 2
    lat = rep * LATTICE
    pos = [(np.asarray(p) + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep)
           for p in POSITIONS]
    Si = dftk.ElementPsp("Si")
    model = dftk.model_DFT(lat, [Si] * len(pos), pos, functionals=dftk.LDA(), symmetries=False,
                           kinetic_blowup=dftk.BlowupCHV())
    basis = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=(1, 1, 1))
    assert basis.kblocks[0].fold_size() > 0
    rho = dftk.guess_density(basis)
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=rho)
    _, ob = _oracle_blocks({}, basis, rho.cpu().numpy(), "CHV", [[0, 0, 0]], [1.0])
    _hpsi_check(basis, ham, ob, lambda ps: [ham[0].mul(ps[0])])
    model = _si_lda(symmetries=False, kinetic_blowup=dftk.BlowupAbinit())
    kc = [[0, 0, 0], [1 / 3, 0, 0], [1 / 3, 1 / 3, 0], [0.1, -0.2, 0.3], [0.5, 0.5, 0]]
    basis = dftk.PlaneWaveBasis(model, Ecut=8, kgrid=dftk.ExplicitKpoints(kc))
    rho = dftk.guess_density(basis)
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=rho)
    _, ob = _oracle_blocks({}, basis, rho.cpu().numpy(), "Abinit", kc, [1 / len(kc)] * len(kc))

    def multi(ps):
        kbs = [ham[ik].bind() for ik in range(len(kc))]
        outs = [torch.empty_like(p) for p in ps]
        dev.apply_h_multi(kbs, ps, outs)
        return outs
    _hpsi_check(basis, ham, ob, multi)


def test_scf_and_direct_minimization_with_blowup():
    """SCF with BlowupCHV against the oracle's SCF with the same table, and direct minimisation (whose preconditioner
    reads the blown-up table) reaching the SCF energy."""
    import dftk_b200 as dftk
    from oracle.basis import Element, Model, PlaneWaveBasis as OBasis
    from oracle import scf as oscf
    model = _si_lda(kinetic_blowup=dftk.BlowupCHV())
    basis = dftk.PlaneWaveBasis(model, Ecut=5, kgrid=(2, 2, 2))
    res = dftk.self_consistent_field(basis, tol=1e-9)
    assert res["converged"]
    std = dftk.self_consistent_field(dftk.PlaneWaveBasis(_si_lda(), Ecut=5, kgrid=(2, 2, 2)), tol=1e-9)
    assert abs(res["energies"]["Kinetic"] - std["energies"]["Kinetic"]) > 1e-6        # the table is in use
    om = Model(LATTICE, [Element("Si")] * 2, POSITIONS)
    with so.extended("CHV"):
        ob = OBasis(om, 5, kgrid=(2, 2, 2))
        ores = oscf.self_consistent_field(ob, tol=1e-9)
    _compare_scf(res, ores, basis, ob, 2, 4)
    dm = dftk.direct_minimization(basis, tol=1e-7)
    assert abs(dm["energies"].total - res["energies"].total) < 1e-8


def test_slab_solve_with_blowup_matches_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29537",
                        os.path.join(ROOT, "scripts", "slab_blowup_check.py")], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("SLAB_BLOWUP_RESULT ")][-1]
    out = json.loads(line[len("SLAB_BLOWUP_RESULT "):])
    assert all(out["converged"]) and out["lobpcg_dlambda"] < 1e-9 and out["dE"] < 1e-8 * out["n_atoms"], out
